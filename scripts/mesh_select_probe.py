"""Time bgs_cloud_select_in_mesh (point-in-mesh selection on the GPU) on the C3 cloud against a 12-triangle box, a
20 480-triangle icosphere and a ~200 k-triangle torus.

    python scripts/mesh_select_probe.py [--reps 20] [--out file.json]

Per mesh: ms per call (CUDA events on the context stream around the synchronous call, after a warm-up call, mean
over --reps calls), the setup / sort / count phases (kernel times from torch.profiler, a separate pass), the inside
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bevy_gaussian_splatting_b200 as B  # noqa: E402
import mesh_cases as MC  # noqa: E402
from select_oracle import select_oracle as SO  # noqa: E402

PHASES = {"mesh_setup_kernel": "setup", "mesh_levels_kernel": "setup", "mesh_emit_kernel": "sort",
          "radix_coop_kernel": "sort", "mesh_count_kernel": "count", "Memset": "clear", "Memcpy": "copy"}


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
            plugin.select_in_mesh(h, *q)
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
        plugin.select_in_mesh(h, *q)                                       # warm-up
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record(stream)
        for _ in range(reps):
            sel = plugin.select_in_mesh(h, *q)
        t1.record(stream)
        t1.synchronize()
        ms = t0.elapsed_time(t1) / reps
        try:
            phases = phase_times(plugin, h, q)
        except Exception as e:   # (the profiler's event API moves between torch releases: keep the timed figure)
            phases = {"unavailable": str(e)[:80]}
        gpu_mask = plugin.visibility(h) == 1.0
        c0 = time.perf_counter()
        cpu_mask, cpu_sel = SO.select_in_mesh(cloud.position_visibility, *q, grid=True)
        cpu_s = time.perf_counter() - c0
    finally:
        h.destroy()
    r = {"mesh": name, "n": len(cloud), "triangles": len(q[1]),
         "gpu_ms_per_call": round(ms, 3), "gpu_phase_ms": {k: round(v, 3) if isinstance(v, float) else v for k, v in sorted(phases.items())},
         "inside": sel, "mask_equals_cpu_grid_oracle": bool(np.array_equal(gpu_mask, cpu_mask)) and sel == cpu_sel,
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
        raise SystemExit("mesh_select_probe: no CUDA device (this probe measures the GPU; there is no CPU figure to give)")
    info = card()
    print(f"card: {info}", flush=True)
    plugin = B.GaussianSplattingPlugin(0)
    rows = []
    c3 = B.random_gaussians_3d_seeded(6_000_000, 0)                    # C3: 6 M f16, seed 0
    lo, hi = np.percentile(c3.position_visibility[:, :3], [20, 80], axis=0)
    c, r = (lo + hi) / 2, float((hi - lo).min()) / 2
    box = MC.box(tuple(lo), tuple(hi))
    ico = MC.icosphere(5, r)
    ico = ((ico[0] + c).astype(np.float32), ico[1])
    tor = MC.torus(316, 316, R=r, r=r * 0.35)
    tor = ((tor[0] + c).astype(np.float32), tor[1])
    for name, mesh in (("box (12 triangles)", box), ("icosphere (20480 triangles)", ico), (f"torus ({len(tor[1])} triangles)", tor)):
        rows.append(probe(plugin, name, c3, mesh, a.reps))
    plugin.destroy()
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"card": info, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
