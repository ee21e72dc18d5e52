"""What a motion-blurred frame costs: one bgs_render_shutter call against what an app does without it -- s
bgs_render_entities_ex calls into RGBA32F premultiplied frames, then a torch mean and sRGB encode -- at 1920x1080 with
s = 2, 4, 8 and 16 samples, on two workloads:

  4d     a 1 M Gaussian4d cloud (random_gaussians_4d_seeded, global_scale 0.02) in time: the samples at
         shutter_times(0.5, 0.2, s) in the window [0, 1], the headless camera
  orbit  bench.py's C3 cloud (6 M seeded gaussians, f16, global_scale 0.02) under an orbiting camera: the samples
         interpolate_view between orbit views 0 and 1 of 120 (a 3-degree arc) at the shutter's midpoints

    python scripts/shutter_probe.py [--frames N] [--out FILE] [--profile]

Both arms write an RGBA8 sRGB 1080p frame to the device.  Before timing, each configuration checks that the shutter's
RGBA32F premultiplied rgb is bit for bit the rule's pairwise mean of the s frames (computed with numpy on the host, in
the rule's order; reported as rule_exact) and that the two arms' RGBA8 frames differ by at most one step.  Then N frames of each arm after 3 of warm-up,
alternated frame by frame (host clock around a call that ends in a device synchronise).  Prints one JSON line: p50 / p90
of each arm, the shutter frame's stage times (bgs_stage_times_us; [4] is the blend and the resolve), libbgs launches,
the sub-frame scratch bytes and the card's name and power limit, read in the same run.  --profile adds the resolve
kernel's time from torch.profiler (a run of its own after the timed frames) and its achieved bandwidth: bytes it must
move (s x 16 B loads and a 4 B store per pixel) over its time, against the H100 SXM's 3.35 TB/s.
"""
from __future__ import annotations

import argparse
import ctypes as C
import dataclasses
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
from scripts.scene_probe import card  # noqa: E402

W, H = 1920, 1080
SAMPLES = (2, 4, 8, 16)
HBM_BYTES_PER_S = 3.35e12


def _pct(ts):
    return {"p50_ms": round(float(np.percentile(ts, 50)) * 1e3, 3), "p90_ms": round(float(np.percentile(ts, 90)) * 1e3, 3)}


def workloads(p):
    """name -> (handle, per-sample (settings, view) of s samples)"""
    c4 = p.add_cloud(B.random_gaussians_4d_seeded(1_000_000, 0))
    st4 = B.CloudSettings(gaussian_mode=B.GaussianMode.Gaussian4d, global_scale=0.02, time_start=0.0, time_stop=1.0)
    head = B.headless_view(W, H)

    def in_time(s):
        return [(dataclasses.replace(st4, time=float(t)), head) for t in B.shutter_times(0.5, 0.2, s)]

    c3 = p.add_cloud(B.random_gaussians_3d_seeded(6_000_000, 0), f16=True)
    st3 = B.CloudSettings(global_scale=0.02)
    a, b = B.orbit_view(0, 120, W, H), B.orbit_view(1, 120, W, H)

    def orbit(s):
        return [(st3, B.interpolate_view(a, b, (i + 0.5) / s)) for i in range(s)]

    return {"4d": (c4, in_time), "orbit": (c3, orbit)}


def pairwise(xs):
    """the rule's sum(0, s) of f32 arrays"""
    if len(xs) == 1:
        return xs[0]
    m = (len(xs) + 1) // 2
    return pairwise(xs[:m]) + pairwise(xs[m:])


def encode_srgb8(c):
    """(H, W, 3) linear f32 -> (H, W, 4) RGBA8 sRGB with alpha 255, as the blend's opaque output"""
    c = c.clamp(0.0, 1.0)
    e = torch.where(c <= 0.0031308, 12.92 * c, 1.055 * c.pow(1.0 / 2.4) - 0.055)
    rgb = (e * 255.0 + 0.5).to(torch.uint8)
    return torch.cat([rgb, torch.full_like(rgb[..., :1], 255)], -1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    res = {"card": card(), "width": W, "height": H, "frames": a.frames}
    p = B.GaussianSplattingPlugin(0)
    lib, ctx = p._lib, p._ctx
    u8, f32 = abi.BGS_FORMAT_RGBA8_SRGB, abi.BGS_FORMAT_RGBA32F

    def check(status):
        if status != abi.BGS_OK:
            raise RuntimeError(lib.bgs_last_error(ctx).decode())

    for name, (h, make) in workloads(p).items():
        for s in SAMPLES:
            smp = make(s)
            st0 = smp[0][0]
            clouds = (C.c_void_p * 1)(h._h.value)
            ents = (abi.bgs_entity_settings * 1)(entity_settings(st0))
            unis = [p.cloud_uniform(st, None, h.aabb) for st, _ in smp]
            all_unis = (abi.bgs_cloud_uniform * s)(*unis)
            one_unis = [(abi.bgs_cloud_uniform * 1)(u) for u in unis]
            vs = (abi.bgs_view * s)(*[v.to_abi() for _, v in smp])
            frame = st0.to_abi()
            premul = st0.to_abi()
            premul.flags |= abi.BGS_FLAG_PREMULTIPLIED_OUT
            out = torch.empty((H, W, 4), dtype=torch.uint8, device="cuda")
            ref = torch.empty_like(out)
            subs = torch.empty((s, H, W, 4), dtype=torch.float32, device="cuda")

            def one(fr=frame, target=out, fmt=u8):
                check(lib.bgs_render_shutter(ctx, clouds, all_unis, ents, None, 1, vs, s, C.byref(fr), None, target.data_ptr(), fmt, 1))

            def each():
                for i in range(s):
                    check(lib.bgs_render_entities_ex(ctx, clouds, one_unis[i], ents, None, 1, C.byref(vs[i]), C.byref(premul), None,
                                                     None, subs[i].data_ptr(), f32, 1))
                ref.copy_(encode_srgb8(subs[..., :3].mean(0)))

            # the rule, and the two arms' frames
            mean32 = torch.empty((H, W, 4), dtype=torch.float32, device="cuda")
            one(premul, mean32, f32)
            each()
            one()
            torch.cuda.synchronize()
            host = subs[..., :3].cpu().numpy()
            want = (pairwise([host[i] for i in range(s)]) / np.float32(s)).astype(np.float32)
            exact = bool(np.array_equal(mean32[..., :3].cpu().numpy(), want))
            step = int((out.int() - ref.int()).abs().max())
            if step > 1:
                raise RuntimeError(f"{name} s={s}: the arms' RGBA8 frames differ by {step} steps")
            for _ in range(3):
                one()
                each()
            torch.cuda.synchronize()
            t1, tn = [], []
            for _ in range(a.frames):
                for arm, ts in ((one, t1), (each, tn)):
                    t0 = time.perf_counter()
                    arm()
                    torch.cuda.synchronize()
                    ts.append(time.perf_counter() - t0)
            one()
            torch.cuda.synchronize()
            stages = [round(float(x), 1) for x in p.stage_times_us()]
            l1 = p.last_launch_count
            check(lib.bgs_render_entities_ex(ctx, clouds, one_unis[0], ents, None, 1, C.byref(vs[0]), C.byref(premul), None, None,
                                             subs[0].data_ptr(), f32, 1))
            ln = p.last_launch_count * s
            fs = p.frame_stats()
            r = {"samples": s, "n": fs.n * s, "rule_exact": exact, "rgba8_max_step": step,
                 "shutter": _pct(t1) | {"launches": l1, "stage_us": stages},
                 "per_sample_calls_torch_mean": _pct(tn) | {"libbgs_launches": ln},
                 "scratch_bytes": s * W * H * 16}
            r["shutter_over_per_sample"] = round(r["shutter"]["p50_ms"] / r["per_sample_calls_torch_mean"]["p50_ms"], 4)
            if a.profile:
                from torch.profiler import ProfilerActivity, profile
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(5):
                        one()
                    torch.cuda.synchronize()
                us, cnt = 0.0, 0
                for e in prof.key_averages():
                    if "shutter_resolve" in e.key:
                        us += float(getattr(e, "self_device_time_total", 0.0) or getattr(e, "self_cuda_time_total", 0.0))
                        cnt += e.count
                if cnt:
                    k_us = us / cnt
                    moved = s * W * H * 16 + W * H * 4
                    r["resolve"] = {"us": round(k_us, 2), "bytes": moved, "GB_per_s": round(moved / (k_us * 1e-6) / 1e9, 1),
                                    "share_of_3_35_TB_per_s": round(moved / (k_us * 1e-6) / HBM_BYTES_PER_S, 3)}
            res[f"{name}_s{s}"] = r
            del subs
            torch.cuda.empty_cache()
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")
    p.destroy()


if __name__ == "__main__":
    main()
