"""Cost of bgs_cloud_transform and bgs_cloud_bounds on the GPU (CUDA events on the context's render stream).

    python scripts/transform_probe.py [--reps 50] [--out FILE]

Clouds: bench.py's 6 M f16 cloud (random_gaussians_3d_seeded(6 M, 0), SH degree 3, 128 B blocks) and a 2 M f32 SH
degree 3 cloud (256 B blocks), each with half of its gaussians selected.  Per cloud and mode: the mean time of one
transform over `reps` back-to-back calls after warm-up, and the bytes it must move over that time, against the H100 SXM's
3.35 TB/s:
    all:      n (2 B + 16)           (read and write every block, write the position plane)
    selected: n B + k (B + 16)       (read every block, write the k selected blocks and their positions)
and the mean time of bgs_cloud_bounds (one pass over the 16 B position plane, then a read-back).  The card's name and
power limit are read in the same run.
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

HBM_BYTES_PER_S = 3.35e12


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return {"nvidia_smi": q[0] if q else "unknown"}


def timed(plugin, fn, reps: int) -> float:
    """Mean milliseconds of fn() over reps calls, between CUDA events on the context's render stream."""
    import torch

    stream = torch.cuda.ExternalStream(plugin.stream_ptr)
    for _ in range(3):
        fn()
    assert plugin.sync()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(reps):
        fn()
    e1.record(stream)
    e1.synchronize()
    assert plugin.sync()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None, help="also write the result as JSON to FILE")
    a = ap.parse_args()
    plugin = B.GaussianSplattingPlugin(0)
    # a rotation about a pivot with a uniform scale of 1 (repeated calls keep the cloud in range)
    M = B.similarity_transform((0.01, 0.0, 0.0), (0.999, 0.02, 0.03, 0.01), 1.0, (1.0, 2.0, 3.0))
    res = {"card": card(), "reps": a.reps, "rows": []}
    for name, n, f16, block in (("6M f16 d3", 6_000_000, True, 128), ("2M f32 d3", 2_000_000, False, 256)):
        c = B.random_gaussians_3d_seeded(n, 0)
        c.position_visibility[:, 3] = (np.arange(n) % 2).astype(np.float32)
        h = plugin.add_cloud(c, f16=f16)
        k = n // 2
        for sel in (False, True):
            ms = timed(plugin, lambda: plugin.transform(h, M, selected=sel), a.reps)
            moved = n * block + k * (block + 16) if sel else n * (2 * block + 16)
            rate = moved / (ms * 1e-3)
            res["rows"].append({"cloud": name, "mode": "selected" if sel else "all", "ms": ms, "bytes": moved,
                                "bytes_per_s": rate, "share_of_3_35_TBps": rate / HBM_BYTES_PER_S})
        t0 = time.perf_counter()
        for _ in range(a.reps):
            plugin.bounds(h)
        bms = (time.perf_counter() - t0) * 1e3 / a.reps
        res["rows"].append({"cloud": name, "mode": "bounds (host clock, includes the read-back)", "ms": bms,
                            "bytes": n * 16, "bytes_per_s": n * 16 / (bms * 1e-3)})
        h.destroy()
    plugin.destroy()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
