"""What a pick frame costs: one bgs_render_entities_pick frame against one bgs_render_entities_ex frame of the same
entities (BGS_FLAG_NO_CHUNKS, the one-round frame a pick frame is), and one bgs_cloud_select_in_view pass, in two scenes:

  c3   bench.py's C3 cloud: 6 M seeded random_gaussians, f16, global_scale 0.02, 1920x1080
  c4   a config-C4-like scene: 2 M seeded 2DGS aabb surfels with a 200 k-gaussian 3DGS object (entities_aux_probe's)

    python scripts/pick_probe.py [--frames N] [--out FILE]

Targets are device memory (rgba8 sRGB and the pick frame).  Each scene first checks that the two colour frames are the
same bytes, then times N frames of each arm after 5 of warm-up, the arms alternated frame by frame (host clock around a
call that ends in a device synchronise).  select_in_view is timed on the C3 cloud with a device mask whose left half is
set.  Prints one JSON line: p50 / p90 of each arm, launch counts, the card's name and power limit.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bevy_gaussian_splatting_b200 as B  # noqa: E402
from bevy_gaussian_splatting_b200 import abi  # noqa: E402
from bevy_gaussian_splatting_b200.plugin import entity_settings  # noqa: E402
from scripts.entities_aux_probe import scene as c4_scene  # noqa: E402
from scripts.scene_probe import card  # noqa: E402


def _pct(ts):
    return {"p50_ms": round(float(np.percentile(ts, 50)) * 1e3, 3), "p90_ms": round(float(np.percentile(ts, 90)) * 1e3, 3)}


def _timed(arms, frames):
    for _ in range(5):
        for f in arms:
            f()
    torch.cuda.synchronize()
    ts = [[] for _ in arms]
    for _ in range(frames):
        for f, t in zip(arms, ts):
            t0 = time.perf_counter()
            f()
            torch.cuda.synchronize()
            t.append(time.perf_counter() - t0)
    return ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pick_probe: no CUDA device")
    res = {"card": card(), "frames": a.frames}
    p = B.GaussianSplattingPlugin(0)
    lib, ctx = p._lib, p._ctx

    def check(status):
        if status != abi.BGS_OK:
            raise RuntimeError(lib.bgs_last_error(ctx).decode())

    c3 = p.add_cloud(B.random_gaussians_3d_seeded(6_000_000, 0), f16=True)
    scenes = {"c3": ([c3], [B.CloudSettings(global_scale=0.02)]), "c4": c4_scene(p)}
    view = B.headless_view(1920, 1080)
    code = abi.BGS_FORMAT_RGBA8_SRGB
    for name, (hs, sts) in scenes.items():
        k = len(hs)
        clouds = (C.c_void_p * k)(*[h._h.value for h in hs])
        unis = (abi.bgs_cloud_uniform * k)(*[p.cloud_uniform(st, None, h.aabb) for h, st in zip(hs, sts)])
        ents = (abi.bgs_entity_settings * k)(*[entity_settings(st) for st in sts])
        s = sts[0].to_abi()
        s.flags = abi.BGS_FLAG_NO_CHUNKS
        v = view.to_abi()
        out = torch.empty((view.height, view.width, 4), dtype=torch.uint8, device="cuda")
        ref = torch.empty_like(out)
        pick = torch.empty((view.height, view.width, 4), dtype=torch.int32, device="cuda")

        def pick_frame():
            check(lib.bgs_render_entities_pick(ctx, clouds, unis, ents, None, k, C.byref(v), C.byref(s), None, None,
                                               out.data_ptr(), code, 1, C.c_void_p(pick.data_ptr())))

        def ex_frame():
            check(lib.bgs_render_entities_ex(ctx, clouds, unis, ents, None, k, C.byref(v), C.byref(s), None, None,
                                             ref.data_ptr(), code, 1))

        pick_frame()
        lp = p.last_launch_count
        ex_frame()
        le = p.last_launch_count
        torch.cuda.synchronize()
        if not torch.equal(out, ref):
            raise RuntimeError(f"{name}: the pick frame's colour differs from bgs_render_entities_ex's")
        tp, te = _timed([pick_frame, ex_frame], a.frames)
        picked = float((pick[..., 0] != -1).float().mean())
        res[name] = {"n": [h.n for h in hs], "bytes_equal": True, "pixels_picked": round(picked, 4),
                     "pick": _pct(tp) | {"launches": lp}, "entities_ex": _pct(te) | {"launches": le}}
        res[name]["pick_over_ex"] = round(res[name]["pick"]["p50_ms"] / res[name]["entities_ex"]["p50_ms"], 4)
    mask = torch.zeros((1080, 1920), dtype=torch.uint8, device="cuda")
    mask[:, :960] = 1
    u = p.cloud_uniform(B.CloudSettings(global_scale=0.02), None, c3.aabb)
    v = view.to_abi()
    inside = C.c_uint32()

    def select():
        check(lib.bgs_cloud_select_in_view(ctx, c3._h, C.byref(u), C.byref(v), C.c_void_p(mask.data_ptr()), 1,
                                           abi.BGS_SELECT_REPLACE, C.byref(inside)))

    (ts,) = _timed([select], a.frames)
    res["select_in_view"] = {"n": c3.n, "inside": inside.value, "mask": "left half of 1920x1080"} | _pct(ts)
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    p.destroy()


if __name__ == "__main__":
    main()
