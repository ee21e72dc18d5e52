"""Time bgs_cloud_subset and bgs_cloud_download_* on the C3 cloud (6 M gaussians, seed 0), f16 and f32.

    python scripts/subset_probe.py [--reps 20] [--out file.json]

Reports, after printing the card's name, power limit and max SM clock (nvidia-smi, read-only), per layout:
  - selection mode with 100 %, 50 % (random) and 1 % (random) of the cloud kept, and index mode with the reversed
    permutation: ms per call (CUDA events on the context stream around each call, mean of --reps after a warm-up);
  - the phases: device time per kernel and copy kind (torch.profiler over the same calls), per call;
  - the algorithmic HBM bytes (selection: the position plane read, the mask words written and read, every kept
    gaussian's 16 B position and its block read and written; index: the index list read plus the same per-gaussian
    copy) and those over the call's time, as a share of the data sheet's 3.35 TB/s;
  - download: ms per call and the bytes delivered to host memory over that time (into freshly allocated numpy
    arrays, as `download_planes` returns them), with the device-to-host copies and the unpack as phases.
"""
from __future__ import annotations

import argparse
import collections
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

import bevy_gaussian_splatting_b200 as B  # noqa: E402

N = 6_000_000
HBM_TBPS = 3.35          # H100 SXM5 80 GB data sheet


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown card (nvidia-smi unavailable)"


def timed(plugin, fn, reps, cleanup=lambda r: None):
    """Mean ms per call (CUDA events on the context stream) and the per-phase device time from torch.profiler.
    cleanup(result) runs after the end event (a subset is destroyed outside the timed span)."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    stream = torch.cuda.ExternalStream(plugin.stream_ptr)
    cleanup(fn())                          # warm-up
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        r = fn()
        b.record(stream)
        b.synchronize()
        ms.append(a.elapsed_time(b))
        cleanup(r)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            cleanup(fn())
        torch.cuda.synchronize()
    phases = collections.defaultdict(float)
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            name = e.name.split("<")[0].split("(")[0].strip()
            phases[name] += e.device_time / 1000.0 / reps
    return float(np.mean(ms)), {k: round(v, 4) for k, v in sorted(phases.items())}


def raw_subset(plugin, h, idx):
    """bgs_cloud_subset alone (the Python handle would also read the positions back for its Aabb)."""
    import ctypes as C

    out, n = C.c_void_p(), C.c_uint32()
    ptr = None if idx is None else idx.ctypes.data_as(C.c_void_p)
    plugin._check(plugin._lib.bgs_cloud_subset(plugin._ctx, h._h, ptr, 0 if idx is None else len(idx), C.byref(out), C.byref(n)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("subset_probe: no CUDA device (this probe measures the GPU)")
    info = card()
    print(f"card: {info}", flush=True)
    plugin = B.GaussianSplattingPlugin(0)
    cloud = B.random_gaussians_3d_seeded(N, 0)
    rng = np.random.default_rng(0)
    rows = []
    for layout in ("f16", "f32"):
        blk = 128 if layout == "f16" else 256
        h = plugin.add_cloud(cloud, f16=layout == "f16")
        for what, frac in (("selection_100", 1.0), ("selection_50", 0.5), ("selection_1", 0.01)):
            plugin.set_visibility(h, (rng.random(N) < frac).astype(np.float32) if frac < 1 else np.ones(N, np.float32))
            kept = int((plugin.visibility(h) >= 0.5).sum())

            ms, ph = timed(plugin, lambda: raw_subset(plugin, h, None), a.reps, plugin._lib.bgs_cloud_destroy)
            byts = N * 16 + 2 * (N // 8) + kept * 2 * (16 + blk)
            rows.append(dict(layout=layout, what=what, kept=kept, ms=round(ms, 4), phases_ms=ph, gb=round(byts / 1e9, 3),
                             tbps=round(byts / ms / 1e9, 3), share=round(byts / ms / 1e9 / HBM_TBPS, 3)))
            print(json.dumps(rows[-1]), flush=True)
        rev = np.arange(N, dtype=np.uint32)[::-1].copy()

        ms, ph = timed(plugin, lambda: raw_subset(plugin, h, rev), a.reps, plugin._lib.bgs_cloud_destroy)
        byts = N * 4 + N * 2 * (16 + blk)
        rows.append(dict(layout=layout, what="index_reversed", kept=N, ms=round(ms, 4), phases_ms=ph, gb=round(byts / 1e9, 3),
                         tbps=round(byts / ms / 1e9, 3), share=round(byts / ms / 1e9 / HBM_TBPS, 3)))
        print(json.dumps(rows[-1]), flush=True)
        ms, ph = timed(plugin, lambda: plugin.download_planes(h), max(3, a.reps // 4))
        host = N * (16 + (96 + 16 if layout == "f16" else 192 + 32))
        rows.append(dict(layout=layout, what="download", kept=N, ms=round(ms, 4), phases_ms=ph, gb=round(host / 1e9, 3),
                         host_gbps=round(host / ms / 1e6, 2)))
        print(json.dumps(rows[-1]), flush=True)
        h.destroy()
    plugin.destroy()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(dict(card=info, n=N, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
