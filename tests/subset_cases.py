"""Visibility lanes for bgs_cloud_subset's selection mode, built to reach every class of its predicate: a gaussian is kept
iff !(w < 0.5f) (include/bgs.h), the set DrawMode::Selected draws.

Classes: 0.5 itself and its f32 neighbours, +-0, +-inf, NaN (both signs, quiet and signalling payloads), subnormals
of both signs, ordinary values on either side, all kept, none kept, and kept / dropped runs that start and end on
either side of the 32-gaussian mask-word and 256-gaussian CTA boundaries of subset.cu."""
from __future__ import annotations

import numpy as np

F = np.float32
HALF = F(0.5)
BELOW_HALF = np.nextafter(HALF, F(0))          # dropped
ABOVE_HALF = np.nextafter(HALF, F(1))          # kept
NAN_BITS = np.array([0x7FC00000, 0xFFC00000, 0x7F800001, 0xFFFFFFFF], np.uint32)   # quiet / negative / signalling
SUBNORMALS = np.array([0x00000001, 0x007FFFFF, 0x80000001, 0x807FFFFF], np.uint32).view(F)

# value -> kept, for every special class
SPECIALS = {
    "half": (HALF, True), "below_half": (BELOW_HALF, False), "above_half": (ABOVE_HALF, True),
    "pos_zero": (F(0.0), False), "neg_zero": (F(-0.0), False), "pos_inf": (F(np.inf), True), "neg_inf": (F(-np.inf), False),
    "one": (F(1.0), True), "neg_one": (F(-1.0), False), "max": (np.finfo(F).max, True), "lowest": (np.finfo(F).min, False),
}
for k, b in enumerate(NAN_BITS):
    SPECIALS[f"nan_{k}"] = (b.view(F), True)
for k, v in enumerate(SUBNORMALS):
    SPECIALS[f"subnormal_{k}"] = (v, False)


def kept(vis: np.ndarray) -> np.ndarray:
    """The rule, restated on the host: !(w < 0.5f)."""
    with np.errstate(invalid="ignore"):
        return ~(np.asarray(vis, F) < HALF)


def runs(n: int, edges) -> np.ndarray:
    """1 / 0 alternating between the sorted `edges`, starting with 1 at 0."""
    v = np.zeros(n, F)
    on, prev = True, 0
    for e in list(edges) + [n]:
        if on:
            v[prev:e] = 1
        on, prev = not on, e
    return v


def cases(scale: int = 1) -> list[dict]:
    """Each case: {name, vis}.  `scale` multiplies the bulk sizes."""
    out = []
    vals = np.array([v for v, _ in SPECIALS.values()], F)
    # every special in every position of a word, cycled through 3 words + 1 (so the last word is partial)
    n = 3 * 32 * len(vals) + 1
    out.append({"name": "specials_cycled", "vis": np.resize(vals, n)})
    # each special alone among dropped and among kept neighbours
    for name, (v, _) in SPECIALS.items():
        a = np.zeros(97, F); a[45] = v
        b = np.ones(97, F); b[45] = v
        out.append({"name": f"{name}_among_dropped", "vis": a})
        out.append({"name": f"{name}_among_kept", "vis": b})
    out.append({"name": "all_kept_1", "vis": np.ones(1, F)})
    out.append({"name": "none_kept_1", "vis": np.zeros(1, F)})
    for m in (31, 32, 33, 255, 256, 257, 1000 * scale):
        out.append({"name": f"all_kept_{m}", "vis": np.full(m, ABOVE_HALF)})
        out.append({"name": f"none_kept_{m}", "vis": np.full(m, BELOW_HALF)})
    # runs straddling mask-word and CTA boundaries
    out.append({"name": "word_edges", "vis": runs(1030, [31, 33, 63, 64, 65, 96, 127, 129, 200, 224, 225, 256, 257, 600])})
    out.append({"name": "cta_edges", "vis": runs(5000, [255, 257, 511, 512, 768, 1023, 1025, 2048, 2304, 4095, 4097])})
    out.append({"name": "first_and_last_only", "vis": np.where(np.arange(2049) % 2048 == 0, F(1), F(0)).astype(F)})
    out.append({"name": "last_only", "vis": np.where(np.arange(4097) == 4096, F(1), F(0)).astype(F)})
    rng = np.random.default_rng(11)
    for p in (0.01, 0.5, 0.99):
        m = 200_000 * scale // 4 + 13
        out.append({"name": f"random_{p}", "vis": (rng.random(m) < p).astype(F)})
    # random mixture of every special value
    out.append({"name": "random_specials", "vis": vals[rng.integers(0, len(vals), 70_001)]})
    return out
