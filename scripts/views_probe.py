"""What several views of one scene cost as one frame: bench.py's C3 room (6 M seeded gaussians, f16, OBB, global_scale
0.02) rendered through one bgs_render_views call and through one bgs_render_entities_ex call per view, in three
configurations:

  stereo  two eyes 64 mm apart at 1920x1080
  cube    six 90-degree 1024x1024 cube faces
  split   four 960x540 split-screen cameras

    python scripts/views_probe.py [--frames N] [--out FILE]

Every view goes to its own device target (rgba8 sRGB).  Each configuration first checks that the two ways give the same
bytes in every view, then times N frames of each after 5 of warm-up, the two arms alternated frame by frame (host clock
around a call that ends in a device synchronise).  Prints one JSON line: p50 and p90 of each arm, the launch counts, the
card's name and power limit.
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
from scripts.scene_probe import card  # noqa: E402

N, SCALE = 6_000_000, 0.02


def configs():
    eye = (0.0, 1.5, 5.0)
    stereo = [B.perspective_view((x, 1.5, 5.0), (x, 1.5, 4.0), 1920, 1080) for x in (-0.032, 0.032)]
    faces = [((1, 0, 0), (0, 1, 0)), ((-1, 0, 0), (0, 1, 0)), ((0, 1, 0), (0, 0, 1)), ((0, -1, 0), (0, 0, 1)),
             ((0, 0, 1), (0, 1, 0)), ((0, 0, -1), (0, 1, 0))]
    cube = [B.perspective_view(eye, tuple(e + d for e, d in zip(eye, dv)), 1024, 1024, fov_y=math.pi / 2, up=up) for dv, up in faces]
    split = [B.perspective_view((x, y, 5.0), (0.0, 1.0, 0.0), 960, 540) for x in (-1.0, 1.0) for y in (1.0, 2.0)]
    return {"stereo": stereo, "cube": cube, "split": split}


def _pct(ts):
    return {"p50_ms": round(float(np.percentile(ts, 50)) * 1e3, 3), "p90_ms": round(float(np.percentile(ts, 90)) * 1e3, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card(), "n": N, "frames": a.frames}
    p = B.GaussianSplattingPlugin(0)
    lib, ctx = p._lib, p._ctx
    st = B.CloudSettings(global_scale=SCALE)
    room = p.add_cloud(B.random_gaussians_3d_seeded(N, 0), f16=True)
    clouds = (C.c_void_p * 1)(room._h.value)
    unis = (abi.bgs_cloud_uniform * 1)(p.cloud_uniform(st, None, room.aabb))
    ents = (abi.bgs_entity_settings * 1)(entity_settings(st))
    s = st.to_abi()
    code = abi.BGS_FORMAT_RGBA8_SRGB

    def check(status):
        if status != abi.BGS_OK:
            raise RuntimeError(lib.bgs_last_error(ctx).decode())

    for name, views in configs().items():
        nv = len(views)
        vs = (abi.bgs_view * nv)(*[v.to_abi() for v in views])
        outs = [torch.empty((v.height, v.width, 4), dtype=torch.uint8, device="cuda") for v in views]
        refs = [torch.empty_like(o) for o in outs]
        targets = (C.c_void_p * nv)(*[o.data_ptr() for o in outs])

        def one():
            check(lib.bgs_render_views(ctx, clouds, unis, ents, None, 1, vs, nv, C.byref(s), None, targets, code, 1))

        def each():
            for i in range(nv):
                check(lib.bgs_render_entities_ex(ctx, clouds, unis, ents, None, 1, C.byref(vs[i]), C.byref(s), None, None,
                                                 refs[i].data_ptr(), code, 1))

        one()
        each()
        torch.cuda.synchronize()
        same = all(torch.equal(o, r) for o, r in zip(outs, refs))
        if not same:
            raise RuntimeError(f"{name}: bgs_render_views and the per-view frames differ")
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
