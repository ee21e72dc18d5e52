"""What the bounding-box overlay (CloudSettings.visualize_bounding_box, BGS_FLAG_VISUALIZE_BOUNDING_BOX) costs on bench.py's
C3 frame (6 M f16 random_gaussians, seed 0, 1920x1080, global_scale 0.02), and on the reference's compare_aabb_obb pair
(the C3 cloud drawn twice side by side through bgs_render_entities_ex, one entity with aabb and one without, both with
the overlay).  One synchronous frame at a time (DESIGN.md §7's frame_ms_p50 convention): p50 / p90 of the frame's CUDA-event
time (key-gen to blend, bgs_stage_times_us; the copy of the frame to the host is outside it) and of the blend stage's,
launches, rounds, pairs and the edge pixel count (alpha exactly 1 in the premultiplied RGBA32F frame).

    python scripts/bbox_probe.py [--frames 60] [--warmup 10] [--out results.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402

import bevy_gaussian_splatting_b200 as B  # noqa: E402
from bevy_gaussian_splatting_b200.plugin import CloudTransform  # noqa: E402


def gpu_facts():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        q = "unknown"
    return q


def timed(pl, fn, frames, warmup):
    rows = []
    for i in range(warmup + frames):
        img = fn()
        if i >= warmup:
            rows.append(pl.stage_times_us())
    st = np.array(rows)
    return img, {"frame_us_p50": float(np.percentile(st[:, 5], 50)), "frame_us_p90": float(np.percentile(st[:, 5], 90)),
                 "blend_us_p50": float(np.percentile(st[:, 4], 50)), "blend_us_p90": float(np.percentile(st[:, 4], 90)),
                 "launches": int(pl.last_launch_count), "rounds": int(pl.frame_stats().rounds),
                 "n_pairs": int(pl.frame_stats().n_pairs)}


def translate(x):
    m = np.eye(4, dtype=np.float32)
    m[0, 3] = x
    return CloudTransform(m)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--n", type=int, default=6_000_000)
    ap.add_argument("--out", default=None, help="also write the results as JSON here")
    a = ap.parse_args()
    cloud = B.random_gaussians_3d_seeded(a.n, 0)
    view = B.headless_view(1920, 1080)
    pl = B.GaussianSplattingPlugin(0)
    h = pl.add_cloud(cloud, f16=True)
    res = {"gpu": gpu_facts(), "workload": f"C3: {a.n} random_gaussians (seed 0), f16, 1920x1080, global_scale 0.02",
           "frames": a.frames, "warmup": a.warmup}
    for name, kw in (("obb", {}), ("aabb", {"aabb": True})):
        for box in (False, True):
            st = B.CloudSettings(global_scale=0.02, visualize_bounding_box=box, **kw)
            img, r = timed(pl, lambda: pl.render_view(h, st, view, fmt="rgba32f", premultiplied=True), a.frames, a.warmup)
            r["edge_pixels"] = int((img[..., 3] == np.float32(1.0)).sum())
            res[f"{name}{'_box' if box else ''}"] = r
            print(name, "box" if box else "plain", json.dumps(r), flush=True)
    # compare_aabb_obb: the cloud twice, side by side, aabb and OBB entities (with and without the overlay)
    for box in (False, True):
        ents = [(h, B.CloudSettings(global_scale=0.02, aabb=True, visualize_bounding_box=box), translate(-12.0)),
                (h, B.CloudSettings(global_scale=0.02, aabb=False, visualize_bounding_box=box), translate(12.0))]
        img, r = timed(pl, lambda: pl.render_entities(ents, view, premultiplied=True), a.frames, a.warmup)
        r["edge_pixels"] = int((img[..., 3] == np.float32(1.0)).sum())
        res[f"compare_aabb_obb{'_box' if box else ''}"] = r
        print("compare_aabb_obb", "box" if box else "plain", json.dumps(r), flush=True)
    pl.destroy()
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
