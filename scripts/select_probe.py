"""Time bgs_cloud_select_sparse (SparseSelect on the GPU) on the C3 cloud, a dense variant of it and a 1 M cloud.

    python scripts/select_probe.py [--reps 20] [--out file.json]

Per cloud: ms per call (CUDA events on the context stream around the synchronous call, after a warm-up call, mean
over --reps calls), the key / sort / count phases (kernel times from torch.profiler, a separate pass), the selected
count, whether the mask equals the CPU grid oracle's, and that oracle's wall time on this host's cores (a CPU number,
labelled as such: it is the reference point, not a GPU measurement).  Prints the card's name and power limit first.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bevy_gaussian_splatting_b200 as B  # noqa: E402
from select_oracle import select_oracle as SO  # noqa: E402

PHASES = {"select_keys_kernel": "key", "radix_coop_kernel": "sort", "select_gather_kernel": "count",
          "select_count_kernel": "count", "Memset": "clear"}


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown card (nvidia-smi unavailable)"


def phase_times(plugin, h, q, calls: int = 5):
    import torch
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            plugin.select_sparse(h, q)
        torch.cuda.synchronize()
    out = {}
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        key = next((v for k, v in PHASES.items() if k in e.name), None)
        if key is None:
            continue
        out[key] = out.get(key, 0.0) + e.device_time / 1000.0 / calls   # us -> ms per call
    return out


def probe(plugin, name, cloud, q, reps):
    import torch

    h = plugin.add_cloud(cloud, f16=True)
    try:
        stream = torch.cuda.ExternalStream(plugin.stream_ptr)
        plugin.select_sparse(h, q)                                         # warm-up
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record(stream)
        for _ in range(reps):
            sel = plugin.select_sparse(h, q)
        t1.record(stream)
        t1.synchronize()
        ms = t0.elapsed_time(t1) / reps
        try:
            phases = phase_times(plugin, h, q)
        except Exception as e:   # (the profiler's event API moves between torch releases: keep the timed figure)
            phases = {"unavailable": str(e)[:80]}
        gpu_mask = plugin.visibility(h) == 1.0
        c0 = time.perf_counter()
        cpu_mask, cpu_sel = SO.select_sparse(cloud.position_visibility, q.radius, q.neighbor_threshold, grid=True)
        cpu_s = time.perf_counter() - c0
    finally:
        h.destroy()
    r = {"cloud": name, "n": len(cloud), "radius": q.radius, "neighbor_threshold": q.neighbor_threshold,
         "gpu_ms_per_call": round(ms, 3), "gpu_phase_ms": {k: round(v, 3) if isinstance(v, float) else v for k, v in sorted(phases.items())},
         "selected": sel, "mask_equals_cpu_grid_oracle": bool(np.array_equal(gpu_mask, cpu_mask)) and sel == cpu_sel,
         "cpu_grid_oracle_s": round(cpu_s, 3), "cpu_threads": os.cpu_count()}
    print(json.dumps(r), flush=True)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("select_probe: no CUDA device (this probe measures the GPU; there is no CPU figure to give)")
    info = card()
    print(f"card: {info}", flush=True)
    plugin = B.GaussianSplattingPlugin(0)
    rows = []
    c3 = B.random_gaussians_3d_seeded(6_000_000, 0)
    rows.append(probe(plugin, "C3 (6M f16, seed 0)", c3, B.SparseSelect(), a.reps))
    dense = B.PlanarGaussian3d(c3.position_visibility.copy(), c3.spherical_harmonic, c3.rotation, c3.scale_opacity)
    dense.position_visibility[:, :3] *= np.float32(0.1)                  # into +-2: tens of neighbours within 0.05
    rows.append(probe(plugin, "C3 dense (positions x0.1, +-2)", dense, B.SparseSelect(), a.reps))
    del c3, dense
    rows.append(probe(plugin, "1M f16 (seed 0)", B.random_gaussians_3d_seeded(1_000_000, 0), B.SparseSelect(), a.reps))
    plugin.destroy()
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"card": info, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
