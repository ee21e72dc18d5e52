"""What loading a large KHR_gaussian_splatting scene costs: a generated 6 M-gaussian SH-3 scene (one primitive, seeded)
written as .glb twice, all-f32 and quantised (i8 normalised rotation, i16 normalised scale, u8 normalised opacity, f32
position and SH), each loaded three ways on the same host:

  gpu      B.load_scene + plugin.add_scene (bgs_cloud_upload_khr: the accessors' spans copied once, decoded on the GPU)
  host     B.load_scene + the CPU decode (khr_oracle) + plugin.add_cloud (bgs_cloud_upload_f32_sh)
  kernel   khr_decode_kernel alone: its device time in torch.profiler (CUDA activity) over one add_scene

    python scripts/khr_probe.py [--n N] [--reps R] [--out FILE]

The .glb files go to a temporary directory.  Each arm's cloud is downloaded and compared byte for byte with the other's
before anything is timed; each arm is then timed R times, alternated (host clock around work that ends in a device
synchronise; the file read is inside the timed window, from the page cache after the first read).  Prints one JSON line:
min / median per arm and format, the kernel time, the card's name and power limit.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile
import time
import warnings

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bevy_gaussian_splatting_b200 as B  # noqa: E402
from khr_cases import A_OP, A_POS, A_ROT, A_SCALE, GltfBuilder, sh_name  # noqa: E402
from khr_oracle import khr_oracle as K  # noqa: E402
from scripts.scene_probe import card  # noqa: E402


def write_scene(path: str, n: int, quantised: bool, seed: int = 0) -> None:
    rng = np.random.default_rng(seed)
    f = np.float32
    arrays = {A_POS: (rng.uniform(-20, 20, (n, 3)).astype(f), False)}
    if quantised:
        arrays[A_ROT] = (rng.integers(-127, 128, (n, 4)).astype(np.int8), True)
        arrays[A_SCALE] = (rng.integers(-32768, -8000, (n, 3)).astype(np.int16), True)
        arrays[A_OP] = (rng.integers(0, 256, (n, 1)).astype(np.uint8), True)
    else:
        arrays[A_ROT] = (rng.uniform(-1, 1, (n, 4)).astype(f), False)
        arrays[A_SCALE] = (rng.uniform(-6, -1, (n, 3)).astype(f), False)
        arrays[A_OP] = (rng.uniform(0, 1, (n, 1)).astype(f), False)
    for k in range(16):
        arrays[sh_name(k)] = (rng.uniform(-1, 1, (n, 3)).astype(f), False)
    b = GltfBuilder()
    names = list(arrays)
    b.node(name="splats", mesh=b.mesh(dict(zip(names, b.accessors_of([arrays[k] for k in names])))))
    with open(path, "wb") as fh:
        fh.write(b.glb())


def gpu_arm(p, path):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        sh = p.add_scene(B.load_scene(path))
    torch.cuda.synchronize()
    return sh.handles[0], sh


def host_arm(p, path):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        cloud, _ = K.decode(B.load_scene(path).primitives[0])
    h = p.add_cloud(cloud)
    torch.cuda.synchronize()
    return h, h


def kernel_ms(path: str) -> float:
    """khr_decode_kernel's own time (torch.profiler, CUDA activity) over one add_scene."""
    from torch.profiler import ProfilerActivity, profile

    p = B.GaussianSplattingPlugin(0)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        scene = B.load_scene(path)
    p.add_scene(scene).destroy()   # warm-up
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        p.add_scene(scene).destroy()
    us = [getattr(e, "self_device_time_total", 0.0) or getattr(e, "self_cuda_time_total", 0.0)
          for e in prof.key_averages() if "khr_decode_kernel" in e.key]
    p.destroy()
    return round(sum(us) / 1e3, 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=6_000_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"n": a.n, "sh_degree": 3, "card": card()}
    p = B.GaussianSplattingPlugin(0)
    with tempfile.TemporaryDirectory() as tmp:
        for quantised in (False, True):
            name = "quantised" if quantised else "f32"
            path = os.path.join(tmp, f"{name}.glb")
            write_scene(path, a.n, quantised)
            r = {"file_mb": round(os.path.getsize(path) / 2**20, 1)}
            hg, og = gpu_arm(p, path)
            hh, oh = host_arm(p, path)
            same = all(np.array_equal(x.view(np.uint32), y.view(np.uint32))
                       for x, y in zip(p.download_planes(hg), p.download_planes(hh)))
            og.destroy(); oh.destroy()
            if not same:
                raise RuntimeError(f"{name}: the GPU decode and the host decode differ")
            times = {"gpu": [], "host": []}
            for _ in range(a.reps):
                for arm, fn in (("gpu", gpu_arm), ("host", host_arm)):
                    t0 = time.perf_counter()
                    _, owner = fn(p, path)
                    times[arm].append((time.perf_counter() - t0) * 1e3)
                    owner.destroy()
            for arm, ts in times.items():
                r[arm] = {"min_ms": round(min(ts), 1), "median_ms": round(float(np.median(ts)), 1)}
            r["bytes_equal"] = same
            r["kernel_ms"] = kernel_ms(path)
            res[name] = r
    p.destroy()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
