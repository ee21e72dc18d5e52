"""Time bgs_cloud_interpolate on the C3 cloud size (6M gaussians, seeds 0 and 1, global_scale 0.02, 1920x1080, as in
bench.py), f16 and f32.

    python scripts/interpolate_probe.py [--reps 100] [--frames 300] [--rounds 4] [--out file.json]

Reports, after printing the card's name and power limit (nvidia-smi, read-only):
  - call_ms per layout: one interpolation alone, CUDA events on the context stream around --reps back-to-back calls
    after a warm-up, mean;
  - the call's algorithmic bytes (f16: two 128 B blocks read, one written, and the 16 B position plane written = 400 B
    per gaussian; f32: two 240 B blocks read, one written (the 16 B pad chunk is neither read nor written), and the
    16 B position plane = 736 B) and that over call_ms, as a share of the data sheet's 3.35 TB/s;
  - frame_ms with and without one interpolation per frame in bench.py's loop (three contexts sharing the f16 cloud,
    consecutive frames alternating between them, every frame queued), --rounds blocks of --frames frames each, the two
    kinds alternating in the same run.  With interpolations, the frame's context queues one into the drawn cloud right
    before its frame, at a time that alternates between 0.25 and 0.75.  Without, the same cloud is drawn as it is.
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
from scripts.particles_probe import HBM_TBPS, card  # noqa: E402

N, W, H, SCALE, IN_FLIGHT = 6_000_000, 1920, 1080, 0.02, 3
BYTES_PER_GAUSSIAN = {"f16": 2 * 128 + 128 + 16, "f32": 2 * 240 + 240 + 16}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=100)
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("interpolate_probe: no CUDA device (this probe measures the GPU)")
    info = card()
    print(f"card: {info}", flush=True)
    plugins = [B.GaussianSplattingPlugin(0) for _ in range(IN_FLIGHT)]
    p0 = plugins[0]
    streams = [torch.cuda.ExternalStream(p.stream_ptr) for p in plugins]
    copy_streams = [torch.cuda.ExternalStream(p.copy_stream_ptr) for p in plugins]
    lc, rc = B.random_gaussians_3d_seeded(N, 0), B.random_gaussians_3d_seeded(N, 1)
    rows = []

    # ---- one call alone, per layout
    clouds = {}
    for layout in ("f32", "f16"):
        hl, hr = p0.add_cloud(lc, f16=layout == "f16"), p0.add_cloud(rc, f16=layout == "f16")
        out = p0.subset(hl, np.arange(N))
        for k in range(10):
            p0.interpolate(out, hl, hr, B.CloudSettings(time=0.25 + 0.5 * (k % 2)))
        assert p0.sync()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record(streams[0])
        for k in range(a.reps):
            p0.interpolate(out, hl, hr, B.CloudSettings(time=0.25 + 0.5 * (k % 2)))
        t1.record(streams[0])
        t1.synchronize()
        ms = t0.elapsed_time(t1) / a.reps
        gb = N * BYTES_PER_GAUSSIAN[layout] / 1e9
        row = {"what": "call", "layout": layout, "gaussians": N, "call_ms": round(ms, 4), "algorithmic_GB": round(gb, 4),
               "GB_per_s": round(gb / (ms / 1e3), 1), "share_of_3.35_TBps": round(gb / (ms / 1e3) / (HBM_TBPS * 1e3), 3)}
        print(json.dumps(row), flush=True)
        rows.append(row)
        if layout == "f16":
            clouds = {"lhs": hl, "rhs": hr, "out": out}
        else:
            out.destroy(); hr.destroy(); hl.destroy()
    del lc, rc

    # ---- bench.py's loop, with and without one interpolation per frame
    hl, hr, out = clouds["lhs"], clouds["rhs"], clouds["out"]
    s = B.CloudSettings(global_scale=SCALE)
    view = B.headless_view(W, H)

    def sync_all():
        ok = True
        for p in plugins:
            ok = p.sync() and ok
        return ok

    def frame(i, with_call):
        p = plugins[i % IN_FLIGHT]
        if with_call:
            p.interpolate(out, hl, hr, B.CloudSettings(time=0.25 + 0.5 * (i % 2)))
        p.render_view(out, s, view, fmt="rgba8_srgb", to_host=False, asynchronous=True)

    def block(with_call):
        for i in range(2 * IN_FLIGHT):
            frame(i, with_call)
        assert sync_all()
        e0 = torch.cuda.Event(enable_timing=True)
        e1 = [torch.cuda.Event(enable_timing=True) for _ in range(2 * IN_FLIGHT)]
        e0.record(streams[0])
        for i in range(a.frames):
            frame(i, with_call)
        for ev, st in zip(e1, streams + copy_streams):
            ev.record(st)
        ok = sync_all()
        return max(e0.elapsed_time(ev) for ev in e1) / a.frames, ok

    for p in plugins:
        p.render_view(out, s, view, fmt="rgba8_srgb", to_host=False)
    block(False)
    block(True)
    loops = {"without_call": [], "with_call": []}
    for r in range(a.rounds):
        for with_call in ((False, True) if r % 2 == 0 else (True, False)):
            ms, ok = block(with_call)
            loops["with_call" if with_call else "without_call"].append(round(ms, 4) if ok else None)
    row2 = {"what": "frame_loop", "contexts": IN_FLIGHT, "frames_per_block": a.frames, "frame_ms": loops,
            "median_without": round(sorted(x for x in loops["without_call"] if x)[len(loops["without_call"]) // 2], 4),
            "median_with": round(sorted(x for x in loops["with_call"] if x)[len(loops["with_call"]) // 2], 4)}
    row2["added_ms_per_frame"] = round(row2["median_with"] - row2["median_without"], 4)
    print(json.dumps(row2), flush=True)
    rows.append(row2)
    out.destroy(); hr.destroy(); hl.destroy()
    for p in plugins:
        p.destroy()
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"card": info, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
