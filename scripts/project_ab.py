"""A/B the projection stage of two libbgs.so builds at bench.py's C3 configuration (6M gaussians, seed 0, f16,
global_scale 0.02, 1920x1080, RGBA8 on the device, three contexts in flight).

    python scripts/project_ab.py --out DIR parent=path/to/libbgs.so new=bevy_gaussian_splatting_b200/libbgs.so

Every build is measured in processes of its own (this script re-invokes itself with --lib), the builds alternating
within each of --repeats rounds, after printing the card's name and power limit (nvidia-smi, read-only).  Per build and
RasterizeMode (Color, Classification, OpticalFlow; scripts/modes_probe.py's settings):
  - stage_us: bgs_stage_times_us of one synchronous frame, median of 20 (index 2 is the projection);
  - frame_ms: bench.py's loop (consecutive frames alternating between three contexts, every frame queued), median of
    3 blocks of 200 frames; CUDA events on every context's streams, the block's time over its frames;
  - kernel_us_in_loop: the projection kernel's mean device time inside that loop, from a torch.profiler pass that runs
    in a process of its own (tracing slows the host, so nothing else is timed there).
The Color frame's records (bgs_debug_projected: front-to-back rank order, 12 words each) and their gaussian ids are
saved as DIR/recs_<tag>.npy and DIR/ids_<tag>.npy; the summary says whether every build's arrays equal the first
build's byte for byte.  Everything printed also goes to DIR/project_ab.json.
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
KERNELS = ("project_kernel", "project_modes_kernel")


def measure(a):
    """One build, one process: the timed figures, or with --profile only the profiler pass."""
    from bevy_gaussian_splatting_b200 import abi

    abi.LIB_PATH = os.path.abspath(a.lib)
    import torch

    import bevy_gaussian_splatting_b200 as B

    if not torch.cuda.is_available():
        raise SystemExit("project_ab: no CUDA device (this probe measures the GPU)")
    modes = {"color": B.RasterizeMode.Color, "classification": B.RasterizeMode.Classification,
             "optical_flow": B.RasterizeMode.OpticalFlow}
    plugins = [B.GaussianSplattingPlugin(0) for _ in range(IN_FLIGHT)]
    streams = [torch.cuda.ExternalStream(p.stream_ptr) for p in plugins]
    copy_streams = [torch.cuda.ExternalStream(p.copy_stream_ptr) for p in plugins]
    h = plugins[0].add_cloud(B.random_gaussians_3d_seeded(N, 0), f16=True)
    plugins[0].set_visibility(h, np.where(np.arange(N) % 2 == 0, 2.0 + (np.arange(N) % 8), 1.0).astype(np.float32))
    view = B.headless_view(W, H)
    eye = np.asarray(view.world_position, np.float64)
    prev = B.perspective_view(tuple(eye + (0.02, -0.01, 0.03)), tuple(eye + (0.02, -0.01, -0.97)), W, H)
    kw = {"previous_view": prev, "delta_time": 1.0 / 60.0}
    settings = {k: B.CloudSettings(global_scale=SCALE, rasterize_mode=m, num_classes=8) for k, m in modes.items()}

    def frame(i, mode, asynchronous=True):
        plugins[i % IN_FLIGHT].render_view(h, settings[mode], view, fmt="rgba8_srgb", to_host=False,
                                           asynchronous=asynchronous, **kw)

    def sync_all():
        ok = True
        for p in plugins:
            ok = p.sync() and ok
        return ok

    def loop(mode, frames):
        for i in range(2 * IN_FLIGHT):
            frame(i, mode)
        assert sync_all()
        e0 = torch.cuda.Event(enable_timing=True)
        e1 = [torch.cuda.Event(enable_timing=True) for _ in range(2 * IN_FLIGHT)]
        e0.record(streams[0])
        for i in range(frames):
            frame(i, mode)
        for ev, st in zip(e1, streams + copy_streams):
            ev.record(st)
        assert sync_all(), "a queued frame overflowed its pair list"
        return max(e0.elapsed_time(ev) for ev in e1) / frames

    row = {"tag": a.tag, "lib": a.lib, "profile": bool(a.profile)}
    for mode in a.modes.split(","):
        for i in range(IN_FLIGHT):
            frame(i, mode, asynchronous=False)
        if a.profile:
            from torch.profiler import ProfilerActivity, profile

            loop(mode, 2 * IN_FLIGHT)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                loop(mode, PROFILED_FRAMES)
                torch.cuda.synchronize()
            t = [e.device_time for e in prof.events()
                 if e.device_type.name == "CUDA" and any(e.name.split("<")[0].endswith(k) for k in KERNELS)]
            row[mode] = {"kernel_us_in_loop": round(float(np.mean(t)), 1), "kernels_seen": len(t)}
            continue
        st = []
        for _ in range(20):
            frame(0, mode, asynchronous=False)
            st.append(plugins[0].stage_times_us())
        row[mode] = {"stage_us": np.median(np.array(st), 0).round(1).tolist(),
                     "n_visible": int(plugins[0].frame_stats().n_visible), "launches": plugins[0].last_launch_count}
        if mode == "color":
            rec, ids = plugins[0].projected()
            np.save(os.path.join(a.out, f"recs_{a.tag}.npy"), rec)
            np.save(os.path.join(a.out, f"ids_{a.tag}.npy"), ids)
        ms = [loop(mode, FRAMES) for _ in range(BLOCKS)]
        row[mode]["frame_ms"] = [round(x, 4) for x in ms]
        row[mode]["frame_ms_median"] = round(float(np.median(ms)), 4)
    h.destroy()
    for p in plugins:
        p.destroy()
    print(json.dumps(row), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("builds", nargs="*", help="tag=path/to/libbgs.so, the reference build first")
    ap.add_argument("--out", required=True)
    ap.add_argument("--repeats", type=int, default=1)
    ap.add_argument("--modes", default="color,classification,optical_flow")
    ap.add_argument("--no-profile", action="store_true", help="skip the torch.profiler processes")
    ap.add_argument("--lib")
    ap.add_argument("--tag")
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    if a.lib:
        return measure(a)
    from scripts.particles_probe import card

    info = card()
    print(f"card: {info}", flush=True)
    builds = [b.split("=", 1) for b in a.builds]
    rows = []
    for rep in range(a.repeats):
        for profile in (False,) if a.no_profile else (False, True):
            for tag, lib in builds:
                cmd = [sys.executable, os.path.abspath(__file__), "--out", a.out, "--lib", lib, "--tag", tag, "--modes", a.modes]
                out = subprocess.run(cmd + (["--profile"] if profile else []), capture_output=True, text=True)
                if out.returncode:
                    raise SystemExit(f"project_ab: {tag} failed\n{out.stdout[-2000:]}\n{out.stderr[-4000:]}")
                rows.append(json.loads(out.stdout.strip().splitlines()[-1]))
                rows[-1]["repeat"] = rep
                print(json.dumps(rows[-1]), flush=True)
    same = {}
    for tag, _ in builds[1:]:
        same[tag] = all(np.load(os.path.join(a.out, f"{k}_{tag}.npy")).tobytes() ==
                        np.load(os.path.join(a.out, f"{k}_{builds[0][0]}.npy")).tobytes() for k in ("recs", "ids"))
    summary = {"what": "records_byte_identical_to_" + builds[0][0], "builds": same}
    print(json.dumps(summary), flush=True)
    with open(os.path.join(a.out, "project_ab.json"), "w") as f:
        json.dump({"card": info, "rows": rows, "summary": summary}, f, indent=1)


if __name__ == "__main__":
    main()
