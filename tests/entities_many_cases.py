"""Inputs of bgs_render_entities_many's tests (tests/test_gpu_entities_many.py, tests/test_host_entities_many.py): a cloud
split into k contiguous pieces whose sizes and boundaries reach key-gen's CTA tiles and phase-2 chunks and the pieces of
1, 31, 32 and 33 gaussians around a warp, and the raw C calls of the capped and uncapped entity frames."""
from __future__ import annotations

import ctypes as C

import numpy as np

from bevy_gaussian_splatting_b200 import abi
from bevy_gaussian_splatting_b200.plugin import entity_settings

KG_TILE = 2048            # keygen.cu: gaussians per key-gen CTA tile (256 threads x 8)
KG_CHUNK = 1024 * 32      # keygen.cu: gaussians per phase-2 chunk (1024 mask words)
SMALL = (1, 31, 32, 33)   # piece sizes around a warp


def split_cuts(n: int, k: int, seed: int = 0) -> list[int]:
    """k + 1 ascending cut points 0 = c_0 < ... < c_k = n: mostly pieces of 1, 31, 32 and 33 gaussians, a few spanning
    several key-gen CTA tiles, and cuts on tile and phase-2 chunk edges where the sizes allow.  Needs n >= 33 k."""
    assert n >= 33 * k, (n, k)
    rng = np.random.default_rng(seed + 31 * k)
    sizes = np.array([SMALL[i % 4] for i in range(k)], np.int64)
    rng.shuffle(sizes)
    spare = n - int(sizes.sum())
    big = rng.choice(k, size=min(k, 8), replace=False)
    share = np.full(len(big), spare // len(big), np.int64)
    share[0] += spare - int(share.sum())
    sizes[big] += share
    cuts = np.concatenate([[0], np.cumsum(sizes)])
    # move a few interior cuts onto tile / chunk edges (keeping every piece non-empty)
    for edge in list(range(KG_TILE, n, KG_TILE))[:: max(1, n // KG_TILE // 16)] + list(range(KG_CHUNK, n, KG_CHUNK)):
        i = int(np.searchsorted(cuts, edge))
        if 0 < i < k and cuts[i - 1] < edge < cuts[i + 1]:
            cuts[i] = edge
    assert cuts[0] == 0 and cuts[-1] == n and (np.diff(cuts) > 0).all()
    return cuts.tolist()


def pieces(n: int, k: int, seed: int = 0) -> list[np.ndarray]:
    cuts = split_cuts(n, k, seed)
    return [np.arange(a, b) for a, b in zip(cuts[:-1], cuts[1:])]


def ok(p, rc):
    assert rc == abi.BGS_OK, p._lib.bgs_last_error(p._ctx)


def error(p) -> str:
    return (p._lib.bgs_last_error(p._ctx) or b"").decode()


def addr(t):
    if t is None:
        return None
    return t.ctypes.data if isinstance(t, np.ndarray) else t.data_ptr()


class Entities:
    """k entities (handles, uniforms, CloudSettings, entity flags) called through bgs_render_entities_ex, _many, _pick or
    _pick_many at `view`, the frame's settings entity 0's without the frame-wide overlay bit, | frame_flags.  The ctypes
    arrays are built once, so a timed call measures the library alone."""

    def __init__(self, p, handles, unis, sts, view, flags=None):
        self.p, self.view, self.k = p, view, len(handles)
        k = self.k
        self.handles, self.sts = list(handles), list(sts)
        self.clouds = (C.c_void_p * k)(*[h._h.value for h in handles])
        self.unis = (abi.bgs_cloud_uniform * k)(*unis)
        self.ents = (abi.bgs_entity_settings * k)(*[entity_settings(st) for st in sts])
        self.flags = (C.c_uint32 * k)(*(flags if flags is not None else [0] * k))
        self.v = view.to_abi()

    def frame(self, frame_flags=0):
        s = self.sts[0].to_abi()
        s.flags = (s.flags & ~abi.BGS_FLAG_VISUALIZE_BOUNDING_BOX) | frame_flags
        return s

    def call(self, name, out, code, frame_flags=0, depth=None, ex=None, device=False, pick=None, k=None, frame=None):
        """bgs_render_entities_<name>'s status (name: ex, many, pick, pick_many); k: the count passed (default all)."""
        s = frame if frame is not None else self.frame(frame_flags)
        zd = None if depth is None else abi.bgs_scene_depth(depth=depth.data_ptr(), pitch_bytes=4 * self.view.width)
        args = [self.p._ctx, self.clouds, self.unis, self.ents, self.flags, self.k if k is None else k, C.byref(self.v),
                C.byref(s), None if ex is None else C.byref(ex), None if zd is None else C.byref(zd), addr(out), code,
                int(device)]
        if name.startswith("pick"):
            args.append(addr(pick))
        return getattr(self.p._lib, "bgs_render_entities_" + name)(*args)
