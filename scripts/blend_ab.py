"""A/B the blend stage of two libbgs.so builds at bench.py's C3 configuration (6M gaussians, seed 0, f16,
global_scale 0.02, 1920x1080, RGBA8 on the device, three contexts in flight).

    python scripts/blend_ab.py --out DIR parent=path/to/libbgs.so new=bevy_gaussian_splatting_b200/libbgs.so

Every build is measured in processes of its own (this script re-invokes itself with --lib), the builds alternating
within each of --repeats rounds, with the card's name, power limit and SM clocks (nvidia-smi, read-only) printed before
and after.  Per build:
  - blend_stage_us: the blend stage of one synchronous frame (bgs_stage_times_us index 4), median of 20;
  - frame_ms: bench.py's loop (consecutive frames alternating between three contexts, every frame queued), median of
    3 blocks of 200 frames; CUDA events on every context's streams, the block's time over its frames;
  - kernel_us_in_loop: the blend kernel's mean device time inside that loop, from a torch.profiler pass that runs in a
    process of its own (tracing slows the host, so nothing else is timed there).
The C3 frame in RGBA8 and RGBA32F and the frame's tile_entries are saved as DIR/<what>_<tag>.npy; the summary says
whether every build's arrays equal the first build's byte for byte.  Everything printed also goes to DIR/blend_ab.json.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N, W, H, SCALE, IN_FLIGHT = 6_000_000, 1920, 1080, 0.02, 3
BLOCKS, FRAMES, PROFILED_FRAMES = 3, 200, 60
KERNELS = ("raster_kernel", "raster2_kernel")
ARRAYS = ("rgba8", "rgba32f", "tile_entries")


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                               "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown card (nvidia-smi unavailable)"


def measure(a):
    """One build, one process: the timed figures, or with --profile only the profiler pass."""
    from bevy_gaussian_splatting_b200 import abi

    abi.LIB_PATH = os.path.abspath(a.lib)
    import torch

    import bevy_gaussian_splatting_b200 as B

    if not torch.cuda.is_available():
        raise SystemExit("blend_ab: no CUDA device (this probe measures the GPU)")
    plugins = [B.GaussianSplattingPlugin(0) for _ in range(IN_FLIGHT)]
    streams = [torch.cuda.ExternalStream(p.stream_ptr) for p in plugins]
    copy_streams = [torch.cuda.ExternalStream(p.copy_stream_ptr) for p in plugins]
    h = plugins[0].add_cloud(B.random_gaussians_3d_seeded(N, 0), f16=True)
    view = B.headless_view(W, H)
    settings = B.CloudSettings(global_scale=SCALE)

    def frame(i, asynchronous=True):
        plugins[i % IN_FLIGHT].render_view(h, settings, view, fmt="rgba8_srgb", to_host=False, asynchronous=asynchronous)

    def sync_all():
        ok = True
        for p in plugins:
            ok = p.sync() and ok
        return ok

    def loop(frames):
        for i in range(2 * IN_FLIGHT):
            frame(i)
        assert sync_all()
        e0 = torch.cuda.Event(enable_timing=True)
        e1 = [torch.cuda.Event(enable_timing=True) for _ in range(2 * IN_FLIGHT)]
        e0.record(streams[0])
        for i in range(frames):
            frame(i)
        for ev, st in zip(e1, streams + copy_streams):
            ev.record(st)
        assert sync_all(), "a queued frame overflowed its pair list"
        return max(e0.elapsed_time(ev) for ev in e1) / frames

    row = {"tag": a.tag, "lib": a.lib, "profile": bool(a.profile)}
    for i in range(IN_FLIGHT):
        frame(i, asynchronous=False)
    if a.profile:
        from torch.profiler import ProfilerActivity, profile

        loop(2 * IN_FLIGHT)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            loop(PROFILED_FRAMES)
            torch.cuda.synchronize()
        t = [e.device_time for e in prof.events()
             if e.device_type.name == "CUDA" and any(e.name.split("<")[0].endswith(k) for k in KERNELS)]
        row["kernel_us_in_loop"] = round(float(np.mean(t)), 1)
        row["kernels_seen"] = len(t)
    else:
        st = []
        for _ in range(20):
            frame(0, asynchronous=False)
            st.append(plugins[0].stage_times_us())
        row["stage_us"] = np.median(np.array(st), 0).round(1).tolist()
        row["blend_stage_us"] = row["stage_us"][4]
        row["launches"] = plugins[0].last_launch_count
        for fmt, code in (("rgba8", "rgba8_srgb"), ("rgba32f", "rgba32f")):
            np.save(os.path.join(a.out, f"{fmt}_{a.tag}.npy"), plugins[0].render_view(h, settings, view, fmt=code))
        np.save(os.path.join(a.out, f"tile_entries_{a.tag}.npy"), plugins[0].tile_entries())
        ms = [loop(FRAMES) for _ in range(BLOCKS)]
        row["frame_ms"] = [round(x, 4) for x in ms]
        row["frame_ms_median"] = round(float(np.median(ms)), 4)
    h.destroy()
    for p in plugins:
        p.destroy()
    print(json.dumps(row), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("builds", nargs="*", help="tag=path/to/libbgs.so, the reference build first")
    ap.add_argument("--out", required=True)
    ap.add_argument("--repeats", type=int, default=1)
    ap.add_argument("--no-profile", action="store_true", help="skip the torch.profiler processes")
    ap.add_argument("--lib")
    ap.add_argument("--tag")
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    if a.lib:
        return measure(a)
    cards = [card()]
    print(f"card: {cards[0]}", flush=True)
    builds = [b.split("=", 1) for b in a.builds]
    rows = []
    for rep in range(a.repeats):
        for profile in (False,) if a.no_profile else (False, True):
            for tag, lib in builds:
                cmd = [sys.executable, os.path.abspath(__file__), "--out", a.out, "--lib", lib, "--tag", tag]
                out = subprocess.run(cmd + (["--profile"] if profile else []), capture_output=True, text=True)
                if out.returncode:
                    raise SystemExit(f"blend_ab: {tag} failed\n{out.stdout[-2000:]}\n{out.stderr[-4000:]}")
                rows.append(json.loads(out.stdout.strip().splitlines()[-1]))
                rows[-1]["repeat"] = rep
                print(json.dumps(rows[-1]), flush=True)
    cards.append(card())
    print(f"card: {cards[1]}", flush=True)
    same = {}
    for tag, _ in builds[1:]:
        same[tag] = {k: np.load(os.path.join(a.out, f"{k}_{tag}.npy")).tobytes() ==
                     np.load(os.path.join(a.out, f"{k}_{builds[0][0]}.npy")).tobytes() for k in ARRAYS}
    summary = {"what": "byte_identical_to_" + builds[0][0], "builds": same}
    print(json.dumps(summary), flush=True)
    with open(os.path.join(a.out, "blend_ab.json"), "w") as f:
        json.dump({"card": cards, "rows": rows, "summary": summary}, f, indent=1)


if __name__ == "__main__":
    main()
