"""Time a frame of RasterizeMode Color, Classification and OpticalFlow at bench.py's C3 configuration (6M gaussians,
seed 0, f16, global_scale 0.02, 1920x1080, RGBA8 on the device, three contexts in flight).

    python scripts/modes_probe.py [--frames 300] [--rounds 4] [--out file.json]

Reports, after printing the card's name and power limit (nvidia-smi, read-only):
  - frame_ms per mode: bench.py's loop (consecutive frames alternating between three contexts, every frame queued),
    --rounds blocks of --frames frames per mode, the three modes rotated within each round; CUDA events on every
    context's streams, the block's wall time over its frames;
  - stage_us per mode: bgs_stage_times_us of one synchronous frame (key-gen, depth sort, projection, binning, tile
    sort, blend), median of 20.
Classification labels one gaussian in two (visibility 2 + i % 8, num_classes 8); OpticalFlow's previous view is the
camera moved by (0.02, -0.01, 0.03) with delta_time 1/60.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bevy_gaussian_splatting_b200 as B  # noqa: E402
from scripts.particles_probe import card  # noqa: E402

N, W, H, SCALE, IN_FLIGHT = 6_000_000, 1920, 1080, 0.02, 3
MODES = {"color": B.RasterizeMode.Color, "classification": B.RasterizeMode.Classification,
         "optical_flow": B.RasterizeMode.OpticalFlow}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("modes_probe: no CUDA device (this probe measures the GPU)")
    info = card()
    print(f"card: {info}", flush=True)
    plugins = [B.GaussianSplattingPlugin(0) for _ in range(IN_FLIGHT)]
    streams = [torch.cuda.ExternalStream(p.stream_ptr) for p in plugins]
    copy_streams = [torch.cuda.ExternalStream(p.copy_stream_ptr) for p in plugins]
    cloud = B.random_gaussians_3d_seeded(N, 0)
    h = plugins[0].add_cloud(cloud, f16=True)
    vis = np.where(np.arange(N) % 2 == 0, 2.0 + (np.arange(N) % 8), 1.0).astype(np.float32)
    plugins[0].set_visibility(h, vis)
    view = B.headless_view(W, H)
    eye = np.asarray(view.world_position, np.float64)
    prev = B.perspective_view(tuple(eye + (0.02, -0.01, 0.03)), tuple(eye + (0.02, -0.01, -0.97)), W, H)
    kw = {"previous_view": prev, "delta_time": 1.0 / 60.0}
    settings = {k: B.CloudSettings(global_scale=SCALE, rasterize_mode=m, num_classes=8) for k, m in MODES.items()}

    def frame(i, mode, asynchronous=True):
        plugins[i % IN_FLIGHT].render_view(h, settings[mode], view, fmt="rgba8_srgb", to_host=False,
                                           asynchronous=asynchronous, **kw)

    def sync_all():
        ok = True
        for p in plugins:
            ok = p.sync() and ok
        return ok

    def block(mode):
        for i in range(2 * IN_FLIGHT):
            frame(i, mode)
        assert sync_all()
        e0 = torch.cuda.Event(enable_timing=True)
        e1 = [torch.cuda.Event(enable_timing=True) for _ in range(2 * IN_FLIGHT)]
        e0.record(streams[0])
        for i in range(a.frames):
            frame(i, mode)
        for ev, st in zip(e1, streams + copy_streams):
            ev.record(st)
        ok = sync_all()
        return max(e0.elapsed_time(ev) for ev in e1) / a.frames, ok

    rows = []
    for mode in MODES:
        for p in plugins:
            p.render_view(h, settings[mode], view, fmt="rgba8_srgb", to_host=False, **kw)
        st = []
        for _ in range(20):
            plugins[0].render_view(h, settings[mode], view, fmt="rgba8_srgb", to_host=False, **kw)
            st.append(plugins[0].stage_times_us())
        row = {"what": "stage_us", "mode": mode, "stage_us": np.median(np.array(st), 0).round(1).tolist(),
               "n_visible": int(plugins[0].frame_stats().n_visible), "launches": plugins[0].last_launch_count}
        print(json.dumps(row), flush=True)
        rows.append(row)
        block(mode)
    loops = {m: [] for m in MODES}
    order = list(MODES)
    for r in range(a.rounds):
        for mode in order[r % 3:] + order[:r % 3]:
            ms, ok = block(mode)
            loops[mode].append(round(ms, 4) if ok else None)
    row = {"what": "frame_loop", "contexts": IN_FLIGHT, "frames_per_block": a.frames, "frame_ms": loops,
           "median": {m: round(float(np.median([x for x in v if x])), 4) for m, v in loops.items()}}
    print(json.dumps(row), flush=True)
    rows.append(row)
    h.destroy()
    for p in plugins:
        p.destroy()
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"card": info, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
