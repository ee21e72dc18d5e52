"""What the G-buffer of several views costs as one frame: a config-C4-like scene (2 M seeded surfels, 2DGS + USE_AABB,
global_scale 0.02, with a 200 k-gaussian 3DGS object in Depth mode inside it) rendered through one bgs_render_views_aux
call and through one bgs_render_entities_aux call per view, in two configurations:

  cube    six 90-degree 1024x1024 cube faces
  stereo  two eyes 64 mm apart at 1920x1080

    python scripts/views_aux_probe.py [--frames N] [--out FILE]

Every view's three frames go to their own device targets (rgba8 sRGB).  Each configuration first checks that the two
ways give the same bytes in every frame of every view, then times N frames of each after 5 of warm-up, the two arms
alternated frame by frame (host clock around a call that ends in a device synchronise).  Prints one JSON line: p50 and
p90 of each arm, the launch counts, the card's name and power limit.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import math
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bevy_gaussian_splatting_b200 as B  # noqa: E402
from bevy_gaussian_splatting_b200 import abi  # noqa: E402
from bevy_gaussian_splatting_b200.plugin import entity_settings  # noqa: E402
from scripts.entities_aux_probe import scene  # noqa: E402
from scripts.scene_probe import card  # noqa: E402


def configs():
    eye = (0.0, 1.5, 5.0)
    faces = [((1, 0, 0), (0, 1, 0)), ((-1, 0, 0), (0, 1, 0)), ((0, 1, 0), (0, 0, 1)), ((0, -1, 0), (0, 0, 1)),
             ((0, 0, 1), (0, 1, 0)), ((0, 0, -1), (0, 1, 0))]
    cube = [B.perspective_view(eye, tuple(e + d for e, d in zip(eye, dv)), 1024, 1024, fov_y=math.pi / 2, up=up) for dv, up in faces]
    stereo = [B.perspective_view((x, 1.5, 5.0), (x, 1.5, 4.0), 1920, 1080) for x in (-0.032, 0.032)]
    return {"cube": cube, "stereo": stereo}


def _pct(ts):
    return {"p50_ms": round(float(np.percentile(ts, 50)) * 1e3, 3), "p90_ms": round(float(np.percentile(ts, 90)) * 1e3, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("views_aux_probe: no CUDA device")
    res = {"card": card(), "frames": a.frames}
    p = B.GaussianSplattingPlugin(0)
    lib, ctx = p._lib, p._ctx
    hs, sts = scene(p)
    sts[1] = B.CloudSettings(rasterize_mode=B.RasterizeMode.Depth)   # (the object over each view's own depth range)
    k = len(hs)
    clouds = (C.c_void_p * k)(*[h._h.value for h in hs])
    unis = (abi.bgs_cloud_uniform * k)(*[p.cloud_uniform(st, None, h.aabb) for h, st in zip(hs, sts)])
    ents = (abi.bgs_entity_settings * k)(*[entity_settings(st) for st in sts])
    s = sts[0].to_abi()
    s.flags = 0
    code = abi.BGS_FORMAT_RGBA8_SRGB
    res["n"] = [h.n for h in hs]

    def check(status):
        if status != abi.BGS_OK:
            raise RuntimeError(lib.bgs_last_error(ctx).decode())

    for name, views in configs().items():
        nv = len(views)
        vs = (abi.bgs_view * nv)(*[v.to_abi() for v in views])
        outs = [[torch.empty((v.height, v.width, 4), dtype=torch.uint8, device="cuda") for _ in range(3)] for v in views]
        refs = [[torch.empty_like(o) for o in trio] for trio in outs]
        targets = [(C.c_void_p * nv)(*[trio[f].data_ptr() for trio in outs]) for f in range(3)]

        def one():
            check(lib.bgs_render_views_aux(ctx, clouds, unis, ents, None, k, vs, nv, C.byref(s), None, *targets, code, 1))

        def each():
            for i in range(nv):
                check(lib.bgs_render_entities_aux(ctx, clouds, unis, ents, None, k, C.byref(vs[i]), C.byref(s), None, None,
                                                  *[r.data_ptr() for r in refs[i]], code, 1))

        one()
        each()
        torch.cuda.synchronize()
        same = all(torch.equal(o, r) for ot, rt in zip(outs, refs) for o, r in zip(ot, rt))
        if not same:
            raise RuntimeError(f"{name}: bgs_render_views_aux and the per-view frames differ")
        for _ in range(5):
            one()
            each()
        torch.cuda.synchronize()
        t1, tv = [], []
        for _ in range(a.frames):
            for arm, ts in ((one, t1), (each, tv)):
                t0 = time.perf_counter()
                arm()
                torch.cuda.synchronize()
                ts.append(time.perf_counter() - t0)
        one()
        l1 = p.last_launch_count
        each()
        lv = p.last_launch_count * nv
        res[name] = {"views": nv, "viewport": [views[0].width, views[0].height], "bytes_equal": same,
                     "one_call": _pct(t1) | {"launches": l1}, "per_view_calls": _pct(tv) | {"launches": lv}}
        res[name]["one_over_per_view"] = round(res[name]["one_call"]["p50_ms"] / res[name]["per_view_calls"]["p50_ms"], 4)
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    p.destroy()


if __name__ == "__main__":
    main()
