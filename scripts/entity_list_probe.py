"""What a frame of a resident entity list costs (bgs_render_entity_list) against bgs_render_entities_many of the same
entities, on entities_many_probe.py's frames:

  (a) bench.py's C3 cloud (6 M seeded gaussians, f16, 1920x1080, global_scale 0.02) split into K = 64, 1 024, 16 384 and
      65 536 contiguous subsets, each an entity with the whole's uniform;
  (b) a 20 k-gaussian object instanced 1 024 and 16 384 times on a grid, half of the instances off-screen.

Each K runs four arms: `many` (bgs_render_entities_many), and the list three ways: `list` (unedited), `list_transforms`
(all K transforms rewritten every frame from a torch CUDA tensor, row-major, before the frame) and `list_set_1pct` (1 %
of the entities set from the host every frame).  The edits write the values the entities already have, so every arm's
frame is the same; each list frame is checked byte for byte against `many` before it is timed, and again after.

    python scripts/entity_list_probe.py [--frames N] [--out FILE]

Per arm: N synchronous frames into a device target after 5 of warm-up, p50 / p90 (host clock around the edit and the
call, ending in a device synchronise), the launch count, the p50 of each stage (bgs_stage_times_us; the expansion runs
before the first stage event, so it shows in the frame time only), and the host return time (p50) of the edit and the
call with BGS_FLAG_ASYNC, which only enqueue.  Prints one JSON line with the card's name and power limit.
"""
from __future__ import annotations

import argparse
import ctypes as C
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
CODE, FLAGS = abi.BGS_FORMAT_RGBA8_SRGB, abi.BGS_FLAG_NO_CHUNKS


class ListArms:
    """The four ways one entity list (EM.Entities) is drawn: `many`, and a bgs_entity_list unedited, with every transform
    rewritten from the device, and with 1 % of the entities set from the host, each frame."""

    def __init__(self, p, ents, view):
        self.p, self.ents, self.view, self.k = p, ents, view, ents.k
        lib = p._lib
        self.h = C.c_void_p()
        EM.ok(p, lib.bgs_entity_list_create(p._ctx, ents.clouds, ents.unis, ents.ents, ents.flags, ents.k, C.byref(self.h)))
        cols = np.array([list(u.transform) for u in ents.unis], np.float32).reshape(-1, 4, 4)
        self.rows = torch.tensor(np.ascontiguousarray(cols.transpose(0, 2, 1)), device="cuda")   # (the uniforms' own values)
        torch.cuda.synchronize()
        count = max(1, self.k // 100)
        idx = [j * (self.k // count) for j in range(count)]
        self.idx = (C.c_uint32 * len(idx))(*idx)
        self.sub = [(C.c_void_p * len(idx))(*[ents.clouds[j] for j in idx]), (abi.bgs_cloud_uniform * len(idx))(*[ents.unis[j] for j in idx]),
                    (abi.bgs_entity_settings * len(idx))(*[ents.ents[j] for j in idx]), (C.c_uint32 * len(idx))(*[ents.flags[j] for j in idx])]
        self.v = view.to_abi()

    def call(self, arm, out, flags=FLAGS):
        p, lib = self.p, self.p._lib
        if arm == "many":
            return self.ents.call("many", out, CODE, flags, device=True)
        if arm == "list_transforms":
            EM.ok(p, lib.bgs_entity_list_set_transforms(self.h, 0, self.k, C.c_void_p(self.rows.data_ptr()), abi.BGS_MATRIX_ROW_MAJOR, 1))
        elif arm == "list_set_1pct":
            EM.ok(p, lib.bgs_entity_list_set(self.h, self.idx, len(self.idx), *self.sub))
        s = self.ents.frame(flags)
        return lib.bgs_render_entity_list(p._ctx, self.h, C.byref(self.v), C.byref(s), None, None, C.c_void_p(out.data_ptr()), CODE, 1)

    def frame(self, arm):
        out = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
        EM.ok(self.p, self.call(arm, out))
        torch.cuda.synchronize()
        return out.cpu().numpy().tobytes()

    def close(self):
        self.p._lib.bgs_entity_list_destroy(self.h)


def arm(lists, name, out, frames):
    p = lists.p
    for _ in range(5):
        EM.ok(p, lists.call(name, out))
    torch.cuda.synchronize()
    ts, stages, host = [], [], []
    for _ in range(frames):
        t0 = time.perf_counter()
        EM.ok(p, lists.call(name, out))
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
        stages.append(p.stage_times_us())
    launches = p.last_launch_count
    for _ in range(min(frames, 20)):
        t0 = time.perf_counter()
        EM.ok(p, lists.call(name, out, FLAGS | abi.BGS_FLAG_ASYNC))
        host.append((time.perf_counter() - t0) * 1e3)
        assert p.sync()
    st = np.percentile(np.array(stages), 50, axis=0)
    return {"k": lists.k, "arm": name, "p50_ms": round(float(np.percentile(ts, 50)), 4),
            "p90_ms": round(float(np.percentile(ts, 90)), 4), "launches": launches,
            "stage_us_p50": [round(float(x), 1) for x in st], "host_call_ms_p50": round(float(np.percentile(host, 50)), 4)}


def run(p, ents, view, out, frames):
    lists = ListArms(p, ents, view)
    want = lists.frame("many")
    rows = []
    for name in ("many", "list", "list_transforms", "list_set_1pct"):
        assert lists.frame(name) == want, f"k = {ents.k}, {name}: the frame differs from many's"
        rows.append(arm(lists, name, out, frames))
        assert lists.frame(name) == want, f"k = {ents.k}, {name}: the frame differs from many's after timing"
    lists.close()
    return rows


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
    for k in (64, 1024, 16384, 65536):
        cuts = np.linspace(0, N, k + 1).astype(np.int64)
        parts = [p.subset(whole, np.arange(lo, hi)) for lo, hi in zip(cuts[:-1], cuts[1:])]
        res["split"] += run(p, EM.Entities(p, parts, [u] * k, [st] * k, view), view, out, a.frames)
        for h in parts:
            h.destroy()
    whole.destroy()
    obj = p.add_cloud(B.random_gaussians_3d_seeded(N_OBJ, 5), f16=True)
    for k in (1024, 16384):
        side = int(np.ceil(np.sqrt(k)))
        trs = []
        for j in range(k):
            gx, gy = j % side, j // side
            m = np.diag([0.05, 0.05, 0.05, 1.0]).astype(np.float32)
            m[:3, 3] = ((gx / side) * 6.0 - 3.0 + (0.0 if gx < side // 2 else 40.0), 1.5 + (gy / side) * 3.0 - 1.5, -2.0)
            trs.append(B.CloudTransform(m))
        res["instanced"] += run(p, EM.Entities(p, [obj] * k, [p.cloud_uniform(st, tr, obj.aabb) for tr in trs], [st] * k, view),
                                view, out, a.frames)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    p.destroy()


if __name__ == "__main__":
    main()
