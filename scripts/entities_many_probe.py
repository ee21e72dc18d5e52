"""What a frame of many entities costs through bgs_render_entities_many (the segment table in device memory):

  (a) bench.py's C3 cloud (6 M seeded gaussians, f16, 1920x1080, global_scale 0.02) whole as one entity, against
      the same cloud split into K = 64, 1 024, 16 384 and 65 536 contiguous subsets, each an entity with the whole's
      uniform (every split frame checked byte for byte against the whole first);
  (b) a 20 k-gaussian object instanced 1 024 and 16 384 times on a grid, half of the instances off-screen;
  (c) bgs_render_entities_many against bgs_render_entities_ex at K = 64 (frames checked byte for byte, launch counts);
  (d) a 1 M-gaussian Gaussian4d cloud (seeded, at time 0.5 of [0, 1]) split into K = 64 subsets through
      bgs_render_entities_ex and _many, and into 1 024 through _many: the 4D projection of the device table
      (project_4d_many_kernel, 3 CTAs per SM) against the by-value one (project_4d_scene_kernel, 4), stage 2 of the times.

    python scripts/entities_many_probe.py [--frames N] [--out FILE]

Each arm: N synchronous frames into a device target after 5 of warm-up, p50 / p90 (host clock around a call that ends
in a device synchronise), the launch count, the p50 of each stage (bgs_stage_times_us: key-gen, depth sort, projection,
binning + tile sort, blend, whole frame), the table bytes copied to the device per frame (the layout api.cu's
many_table stages: 344 B SceneSeg, 4 B offset, 12 B times, 4 B num_classes, 4 B kind per entity, each region padded to
256 B; 0 for the capped calls, whose table is a kernel parameter), and the host time of the call (p50 of the return
time of the same call with BGS_FLAG_ASYNC, which only enqueues).  Prints one JSON line with the card's name and power
limit beside the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bevy_gaussian_splatting_b200 as B  # noqa: E402
import entities_many_cases as EM  # noqa: E402
from bevy_gaussian_splatting_b200 import abi  # noqa: E402
from scripts.scene_probe import card  # noqa: E402

W, H, N, SCALE = 1920, 1080, 6_000_000, 0.02
N_OBJ = 20_000
N_4D = 1_000_000


def table_bytes(k: int) -> int:
    pad = lambda b: (b + 255) // 256 * 256   # noqa: E731
    return sum(pad(k * s) for s in (344, 4, 12, 4, 4))


def arm(p, ents, name, out, frames, k):
    code = abi.BGS_FORMAT_RGBA8_SRGB
    for _ in range(5):
        EM.ok(p, ents.call(name, out, code, abi.BGS_FLAG_NO_CHUNKS, device=True))
    torch.cuda.synchronize()
    ts, stages, host = [], [], []
    for _ in range(frames):
        t0 = time.perf_counter()
        EM.ok(p, ents.call(name, out, code, abi.BGS_FLAG_NO_CHUNKS, device=True))
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
        stages.append(p.stage_times_us())
    launches = p.last_launch_count
    for _ in range(min(frames, 20)):
        t0 = time.perf_counter()
        EM.ok(p, ents.call(name, out, code, abi.BGS_FLAG_NO_CHUNKS | abi.BGS_FLAG_ASYNC, device=True))
        host.append((time.perf_counter() - t0) * 1e3)
        assert p.sync()
    st = np.percentile(np.array(stages), 50, axis=0)
    return {"k": k, "call": name, "p50_ms": round(float(np.percentile(ts, 50)), 4), "p90_ms": round(float(np.percentile(ts, 90)), 4),
            "launches": launches, "stage_us_p50": [round(float(x), 1) for x in st],
            "table_bytes": table_bytes(k) if name == "many" else 0, "host_call_ms_p50": round(float(np.percentile(host, 50)), 4)}


def frame_bytes(p, ents, name):
    out = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
    EM.ok(p, ents.call(name, out, abi.BGS_FORMAT_RGBA8_SRGB, abi.BGS_FLAG_NO_CHUNKS, device=True))
    torch.cuda.synchronize()
    return out.cpu().numpy().tobytes()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=30)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card(), "n": N, "viewport": [W, H], "frames": a.frames, "split": [], "instanced": []}
    p = B.GaussianSplattingPlugin(0)
    view = B.headless_view(W, H)
    st = B.CloudSettings(global_scale=SCALE)
    whole = p.add_cloud(B.random_gaussians_3d_seeded(N, 0), f16=True)
    u = p.cloud_uniform(st, None, whole.aabb)
    out = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
    one = EM.Entities(p, [whole], [u], [st], view)
    want = frame_bytes(p, one, "many")
    res["whole"] = arm(p, one, "ex", out, a.frames, 1)
    for k in (64, 1024, 16384, 65536):
        cuts = np.linspace(0, N, k + 1).astype(np.int64)
        parts = [p.subset(whole, np.arange(lo, hi)) for lo, hi in zip(cuts[:-1], cuts[1:])]
        ents = EM.Entities(p, parts, [u] * k, [st] * k, view)
        assert frame_bytes(p, ents, "many") == want, f"split into {k}: frame differs from the whole"
        if k == 64:   # (c)
            assert frame_bytes(p, ents, "ex") == want
            res["ex_64"] = arm(p, ents, "ex", out, a.frames, k)
        res["split"].append(arm(p, ents, "many", out, a.frames, k))
        for h in parts:
            h.destroy()
    whole.destroy()
    obj = p.add_cloud(B.random_gaussians_3d_seeded(N_OBJ, 5), f16=True)
    ost = B.CloudSettings(global_scale=SCALE)
    for k in (1024, 16384):
        side = int(np.ceil(np.sqrt(k)))
        trs = []
        for j in range(k):
            gx, gy = j % side, j // side
            m = np.diag([0.05, 0.05, 0.05, 1.0]).astype(np.float32)
            # columns beyond the grid's first half sit far to the right of the view: half the instances off-screen
            m[:3, 3] = ((gx / side) * 6.0 - 3.0 + (0.0 if gx < side // 2 else 40.0), 1.5 + (gy / side) * 3.0 - 1.5, -2.0)
            trs.append(B.CloudTransform(m))
        ents = EM.Entities(p, [obj] * k, [p.cloud_uniform(ost, tr, obj.aabb) for tr in trs], [ost] * k, view)
        r = arm(p, ents, "many", out, a.frames, k)
        r["n_visible"] = int(p.frame_stats().n_visible)
        res["instanced"].append(r)
    st4 = B.CloudSettings(global_scale=SCALE, gaussian_mode=B.GaussianMode.Gaussian4d, time=0.5, time_start=0.0, time_stop=1.0)
    perf = p.add_cloud(B.random_gaussians_4d_seeded(N_4D, 3))
    u4 = p.cloud_uniform(st4, None, perf.aabb)
    res["gaussian4d"] = []
    for k, calls in ((64, ("ex", "many")), (1024, ("many",))):
        cuts = np.linspace(0, N_4D, k + 1).astype(np.int64)
        parts = [p.subset(perf, np.arange(lo, hi)) for lo, hi in zip(cuts[:-1], cuts[1:])]
        ents = EM.Entities(p, parts, [u4] * k, [st4] * k, view)
        if k == 64:
            assert frame_bytes(p, ents, "ex") == frame_bytes(p, ents, "many"), "4D split into 64: _many differs from _ex"
        for name in calls:
            res["gaussian4d"].append(arm(p, ents, name, out, a.frames, k))
        for h in parts:
            h.destroy()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    p.destroy()


if __name__ == "__main__":
    main()
