"""Cost of bgs_render_entities_aux: one colour + depth + normal pass over a scene vs the three bgs_render_entities_ex frames
it replaces (as given, every entity in Depth, every entity in Normal).

The scene: config C4's cloud (2M surfels, 2DGS + USE_AABB) as a room scan, with a 200k-gaussian 3DGS object (quad-uv)
inside it, 1920x1080, RGBA8 device targets; with and without a depth buffer.  Both arms are synchronous calls timed with
a host clock (each returns after its stream synchronises), warmed up, then alternated in one process; the spread is the
min / max over the timed rounds.  The three aux frames are checked against the three _ex frames byte for byte first.

    python scripts/entities_aux_probe.py [--rounds 30] [--out results.json]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np
import torch

import bevy_gaussian_splatting_b200 as B
from bevy_gaussian_splatting_b200 import abi
from bevy_gaussian_splatting_b200.plugin import entity_settings

W, H = 1920, 1080


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    name, power, clock = [x.strip() for x in q.split(",")] if q.count(",") == 2 else (q, "?", "?")
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def scene(p):
    room = B.random_gaussians_3d_seeded(2_000_000, 4)   # (aux_probe.py's config C4 cloud)
    obj = B.random_gaussians_3d_seeded(200_000, 7)
    pos = obj.position_visibility.copy()
    pos[:, :3] *= np.float32(0.1)
    so = obj.scale_opacity.copy()
    so[:, :3] *= np.float32(0.1)
    obj = B.PlanarGaussian3d(pos, obj.spherical_harmonic, obj.rotation, so)
    hs = [p.add_cloud(room), p.add_cloud(obj)]
    sts = [B.CloudSettings(global_scale=0.02, gaussian_mode=B.GaussianMode.Gaussian2d, aabb=True), B.CloudSettings()]
    return hs, sts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the result as JSON to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("entities_aux_probe: no CUDA device")
    p = B.GaussianSplattingPlugin(0)
    hs, sts = scene(p)
    k = len(hs)
    clouds = (C.c_void_p * k)(*[h._h.value for h in hs])
    unis = (abi.bgs_cloud_uniform * k)(*[p.cloud_uniform(st, None, h.aabb) for h, st in zip(hs, sts)])
    view = B.headless_view(W, H).to_abi()
    frame = sts[0].to_abi()
    frame.flags = 0

    def ents(mode=None):
        return (abi.bgs_entity_settings * k)(*[entity_settings(st if mode is None else
                                                               B.CloudSettings(**{**vars(st), "rasterize_mode": mode}))
                                               for st in sts])

    given, as_depth, as_normal = ents(), ents(B.RasterizeMode.Depth), ents(B.RasterizeMode.Normal)
    outs = [torch.empty((H, W, 4), dtype=torch.uint8, device="cuda") for _ in range(3)]
    exs = [torch.empty((H, W, 4), dtype=torch.uint8, device="cuda") for _ in range(3)]
    depth_buf = torch.rand((H, W), generator=torch.Generator(device="cuda").manual_seed(1), device="cuda") * 0.04
    result = {"card": card(), "scene": "2M-surfel 2DGS aabb room + 200k 3DGS OBB object, 1920x1080, rgba8 device targets",
              "rounds": a.rounds, "warmup": a.warmup, "arms": {}}

    for label, zd in (("no depth buffer", None), ("depth buffer", abi.bgs_scene_depth(depth=depth_buf.data_ptr(), pitch_bytes=4 * W))):
        zp = None if zd is None else C.byref(zd)

        def aux():
            p._check(p._lib.bgs_render_entities_aux(p._ctx, clouds, unis, given, None, k, C.byref(view), C.byref(frame), None, zp,
                                                    *[o.data_ptr() for o in outs], abi.BGS_FORMAT_RGBA8_SRGB, 1))

        def three():
            for e, o in zip((given, as_depth, as_normal), exs):
                p._check(p._lib.bgs_render_entities_ex(p._ctx, clouds, unis, e, None, k, C.byref(view), C.byref(frame), None, zp,
                                                       o.data_ptr(), abi.BGS_FORMAT_RGBA8_SRGB, 1))

        aux(); three()
        torch.cuda.synchronize()
        same = all(torch.equal(x, y) for x, y in zip(outs, exs))
        fs = p.frame_stats()
        t = {"aux": [], "three": []}
        for r in range(a.warmup + a.rounds):
            for name, fn in (("aux", aux), ("three", three)) if r % 2 == 0 else (("three", three), ("aux", aux)):
                t0 = time.perf_counter()
                fn()
                dt = (time.perf_counter() - t0) * 1e3
                if r >= a.warmup:
                    t[name].append(dt)
        row = {"frames_identical": same, "n_visible": fs.n_visible, "n_pairs": fs.n_pairs}
        for name, v in t.items():
            v = np.array(v)
            row[name] = {"median_ms": float(np.median(v)), "min_ms": float(v.min()), "max_ms": float(v.max())}
        row["aux_over_three"] = row["aux"]["median_ms"] / row["three"]["median_ms"]
        result["arms"][label] = row
        print(f"{label}: aux {row['aux']['median_ms']:.2f} ms [{row['aux']['min_ms']:.2f}, {row['aux']['max_ms']:.2f}]  "
              f"three _ex {row['three']['median_ms']:.2f} ms [{row['three']['min_ms']:.2f}, {row['three']['max_ms']:.2f}]  "
              f"ratio {row['aux_over_three']:.3f}  identical={same}  n_vis={fs.n_visible} pairs={fs.n_pairs}")
    print(json.dumps(result))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)
    p.destroy()


if __name__ == "__main__":
    main()
