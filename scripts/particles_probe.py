"""Time bgs_cloud_particles_step on the C3 cloud (6M f16, seed 0, global_scale 0.02, 1920x1080, as in bench.py) with
random_particle_behaviors(6_000_000, 0).

    python scripts/particles_probe.py [--reps 100] [--frames 300] [--rounds 4] [--out file.json]

Reports, after printing the card's name and power limit (nvidia-smi, read-only):
  - step_ms: one step alone, CUDA events on the context stream around --reps back-to-back steps after a warm-up, mean;
  - the step's algorithmic bytes (144 B per active behaviour: the 64 B record and the 16 B position read, the 16 B
    position written twice and the 32 B of velocity and acceleration written) and that over step_ms, as a share of
    the data sheet's 3.35 TB/s;
  - frame_ms with and without one step per frame in bench.py's loop (three contexts sharing the cloud, consecutive
    frames alternating between them, every frame queued), --rounds blocks of --frames frames each, the two kinds
    alternating in the same run.  With steps, the frame's context queues the step right before its frame, with dt
    alternating +1/60 and -1/60 so the cloud stays where the frames without steps see it.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bevy_gaussian_splatting_b200 as B  # noqa: E402

N, W, H, SCALE, IN_FLIGHT = 6_000_000, 1920, 1080, 0.02, 3
HBM_TBPS = 3.35          # H100 SXM5 80 GB data sheet
BYTES_PER_BEHAVIOUR = 144


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown card (nvidia-smi unavailable)"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=100)
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("particles_probe: no CUDA device (this probe measures the GPU)")
    info = card()
    print(f"card: {info}", flush=True)
    plugins = [B.GaussianSplattingPlugin(0) for _ in range(IN_FLIGHT)]
    cloud = B.random_gaussians_3d_seeded(N, 0)
    h = plugins[0].add_cloud(cloud, f16=True)
    beh = B.random_particle_behaviors(N, 0)
    parts = plugins[0].add_particles(beh)
    active = int((beh["indices"][:, 0] < 0x80000000).sum())
    del cloud, beh
    streams = [torch.cuda.ExternalStream(p.stream_ptr) for p in plugins]
    copy_streams = [torch.cuda.ExternalStream(p.copy_stream_ptr) for p in plugins]
    s = B.CloudSettings(global_scale=SCALE)
    view = B.headless_view(W, H)

    # ---- the step alone
    p0 = plugins[0]
    for k in range(10):
        p0.step_particles(h, parts, 1 / 60 if k % 2 == 0 else -1 / 60)
    assert p0.sync()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record(streams[0])
    for k in range(a.reps):
        p0.step_particles(h, parts, 1 / 60 if k % 2 == 0 else -1 / 60)
    t1.record(streams[0])
    t1.synchronize()
    step_ms = t0.elapsed_time(t1) / a.reps
    gb = active * BYTES_PER_BEHAVIOUR / 1e9
    row = {"what": "step", "behaviours": active, "step_ms": round(step_ms, 4), "algorithmic_GB": round(gb, 4),
           "GB_per_s": round(gb / (step_ms / 1e3), 1), "share_of_3.35_TBps": round(gb / (step_ms / 1e3) / (HBM_TBPS * 1e3), 3)}
    print(json.dumps(row), flush=True)

    # ---- bench.py's loop, with and without one step per frame
    def sync_all():
        ok = True
        for p in plugins:
            ok = p.sync() and ok
        return ok

    def frame(i, with_step):
        p = plugins[i % IN_FLIGHT]
        if with_step:
            p.step_particles(h, parts, 1 / 60 if i % 2 == 0 else -1 / 60)
        p.render_view(h, s, view, fmt="rgba8_srgb", to_host=False, asynchronous=True)

    def block(with_step):
        for i in range(2 * IN_FLIGHT):
            frame(i, with_step)
        assert sync_all()
        e0 = torch.cuda.Event(enable_timing=True)
        e1 = [torch.cuda.Event(enable_timing=True) for _ in range(2 * IN_FLIGHT)]
        e0.record(streams[0])
        for i in range(a.frames):
            frame(i, with_step)
        for ev, st in zip(e1, streams + copy_streams):
            ev.record(st)
        ok = sync_all()
        return max(e0.elapsed_time(ev) for ev in e1) / a.frames, ok

    for p in plugins:
        p.render_view(h, s, view, fmt="rgba8_srgb", to_host=False)
    block(False)
    block(True)
    loops = {"without_step": [], "with_step": []}
    for r in range(a.rounds):
        for with_step in ((False, True) if r % 2 == 0 else (True, False)):
            ms, ok = block(with_step)
            loops["with_step" if with_step else "without_step"].append(round(ms, 4) if ok else None)
    row2 = {"what": "frame_loop", "contexts": IN_FLIGHT, "frames_per_block": a.frames, "frame_ms": loops,
            "median_without": round(sorted(x for x in loops["without_step"] if x)[len(loops["without_step"]) // 2], 4),
            "median_with": round(sorted(x for x in loops["with_step"] if x)[len(loops["with_step"]) // 2], 4)}
    row2["added_ms_per_frame"] = round(row2["median_with"] - row2["median_without"], 4)
    print(json.dumps(row2), flush=True)
    parts.destroy()
    h.destroy()
    for p in plugins:
        p.destroy()
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"card": info, "rows": [row, row2]}, f, indent=1)


if __name__ == "__main__":
    main()
