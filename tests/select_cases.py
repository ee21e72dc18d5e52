"""Inputs for the SparseSelect tests (CPU oracle and GPU): cloud generators, knife-edge pairs, and a restatement of
the hashed grid's cell / bucket functions (bevy_gaussian_splatting_b200/csrc/select.cu) to build inputs that reach
the grid's corner cases on purpose."""
from __future__ import annotations

import math

import numpy as np

# ---- the rule, restated in numpy float32 (written from include/bgs.h, not from the oracle) ----------------------------


def numpy_select(pos_vis: np.ndarray, radius: float, threshold: int) -> np.ndarray:
    """count_i = #{j : ((dx*dx + dy*dy) + dz*dz) < r2}, dx = x_j - x_i, f32 throughout; selected iff count < threshold."""
    p = np.ascontiguousarray(pos_vis[:, :3], np.float32)
    n = len(p)
    r2 = np.float32(radius) * np.float32(radius)
    cnt = np.zeros(n, np.int64)
    with np.errstate(invalid="ignore", over="ignore"):
        for lo in range(0, n, 256):
            d = p[None, :, :] - p[lo:lo + 256, None, :]          # [i, j] = p_j - p_i
            sq = d * d
            d2 = (sq[..., 0] + sq[..., 1]) + sq[..., 2]
            cnt[lo:lo + 256] = (d2 < r2).sum(1)
    return cnt < threshold


def d2_f32(a, b) -> np.float32:
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    d = (b - a).astype(np.float32)
    sq = (d * d).astype(np.float32)
    return np.float32(np.float32(sq[..., 0] + sq[..., 1]) + sq[..., 2])


# ---- clouds ---------------------------------------------------------------------------------------------------------


def pos_cloud(xyz: np.ndarray) -> np.ndarray:
    out = np.ones((len(xyz), 4), np.float32)
    out[:, :3] = xyz
    return out


def uniform(n: int, seed: int, half: float = 20.0) -> np.ndarray:
    rng = np.random.default_rng(seed)
    return pos_cloud(rng.uniform(-half, half, (n, 3)).astype(np.float32))


def clustered(n: int, seed: int, clusters: int = 64, sigma: float = 0.05, half: float = 20.0) -> np.ndarray:
    """Gaussian blobs (dense) plus 10 % uniform background (sparse floaters)."""
    rng = np.random.default_rng(seed)
    centres = rng.uniform(-half, half, (clusters, 3))
    nb = n // 10
    which = rng.integers(0, clusters, n - nb)
    xyz = np.concatenate([centres[which] + rng.normal(0, sigma, (n - nb, 3)), rng.uniform(-half, half, (nb, 3))])
    return pos_cloud(rng.permutation(xyz).astype(np.float32))


def with_duplicates(n: int, seed: int) -> np.ndarray:
    p = uniform(n, seed, 2.0)
    rng = np.random.default_rng(seed + 1)
    src = rng.integers(0, n, n // 3)
    dst = rng.integers(0, n, n // 3)
    p[dst] = p[src]                                               # exact repeats, some several times
    p[: min(n, 40), :3] = p[0, :3]                                 # one position 40 times
    return p


def non_finite(n: int, seed: int) -> np.ndarray:
    p = uniform(n, seed, 2.0)
    bad = [np.nan, np.inf, -np.inf]
    for k in range(0, n, 7):
        p[k, k % 3] = bad[(k // 7) % 3]
    return p


def large_coordinates(n: int, seed: int) -> np.ndarray:
    """Coordinates up to 1e6 (f32 ulp 0.0625 there): exact duplicates and ulp-adjacent neighbours at large
    magnitude, for radius 1e-3 -- cell coordinates near 1e9, the hash and clamp path."""
    rng = np.random.default_rng(seed)
    base = rng.uniform(-1e6, 1e6, (n // 4, 3)).astype(np.float32)
    reps = base[rng.integers(0, len(base), n - len(base))].copy()
    step = rng.integers(0, 2, reps.shape).astype(np.int32) * rng.choice([-1, 1], reps.shape).astype(np.int32)
    reps = (reps.view(np.int32) + step).view(np.float32)           # same value or one ulp apart
    small = rng.uniform(-1e-2, 1e-2, (n // 8, 3)).astype(np.float32)
    xyz = np.concatenate([base, reps[: n - len(base) - len(small)], small])
    return pos_cloud(rng.permutation(xyz))


# ---- knife-edge pairs: d2 == r2 exactly, one ulp below, one ulp above ------------------------------------------------

EDGE_KINDS = ("equal", "below", "above")


def _targets(radius: float):
    r2 = np.float32(radius) * np.float32(radius)
    return {"equal": r2, "below": np.nextafter(r2, np.float32(0)), "above": np.nextafter(r2, np.float32(np.inf))}


def _ulps(x: float, k: int) -> np.ndarray:
    v = np.float32(x)
    return (np.array([v]).view(np.int32) + np.arange(-k, k + 1, dtype=np.int32)).view(np.float32)


def _cell(p: float, radius: float) -> int:
    q = float(np.float64(np.float32(p))) / (float(np.float32(radius)) * (1.0 + 1.0 / 1024.0))
    return math.floor(max(-2.0 ** 40, min(2.0 ** 40, q)))


def _edge_search(radius: float, geo: str, x0: float):
    """Pairs (p_i, p_j) near the origin hitting the three targets, for one geometry and one start x0.  Coordinates stay
    of the order of the radius, so one ulp of a coordinate moves d2 by about one ulp of r2.  The offset that separates
    pairs goes into a coordinate both points share, whose difference is exactly 0."""
    t = _targets(radius)
    r = float(np.float32(radius))
    xi = np.float32(x0)
    if geo == "boundary":
        # x_i: the largest f32 below a cell boundary, x_j ~ x_i + r in the next cell
        k = _cell(x0, radius) + 1
        xi = max(x for x in _ulps(k * r * (1.0 + 1.0 / 1024.0), 8) if _cell(x, radius) == k - 1)
    pi = np.array([xi, xi if geo == "diagonal" else 0.0, 0.0], np.float32)
    if geo == "diagonal":
        h = r / math.sqrt(2.0)
        cand = np.stack(np.meshgrid(_ulps(float(xi) + h, 40), _ulps(float(xi) + h, 40), indexing="ij"), -1).reshape(-1, 2)
        pj = np.concatenate([cand, np.zeros((len(cand), 1), np.float32)], 1)
    else:
        xs = _ulps(float(xi) + r, 400)
        pj = np.stack([xs, np.zeros(len(xs), np.float32), np.zeros(len(xs), np.float32)], 1)
    d2 = d2_f32(pi[None, :], pj)
    out = {}
    for kind in EDGE_KINDS:
        hit = np.flatnonzero(d2 == t[kind])
        if len(hit):
            out[kind] = (pi, pj[hit[0]].astype(np.float32))
    return out


def _edge_cloud_at(radius: float):
    pts, where = [], {}
    r = float(np.float32(radius))
    for geo in ("axis", "diagonal", "boundary"):
        for x0 in (0.0, 0.37 * r, 1.3 * r, 2.9 * r, 5.1 * r):
            for kind, (pi, pj) in _edge_search(radius, geo, x0).items():
                if (geo, kind) in where:
                    continue
                off = np.zeros(3, np.float32)
                off[2 if geo == "diagonal" else 1] = 16.0 * (1 + len(where))   # (shared coordinate: difference 0)
                where[(geo, kind)] = (len(pts), len(pts) + 1)
                pts += [pi + off, pj + off]
    return pos_cloud(np.array(pts, np.float32).reshape(-1, 3)), where


def knife_edge_cloud(radius: float):
    """One pair per (geometry, kind), geometry in axis / diagonal / boundary (an axis pair whose two points lie in
    different cells), kind in EDGE_KINDS, 16 units apart from the next pair.  On an axis d2 = fl(dx * dx) over the f32
    values of dx near the radius, which step d2 by about 2 * mantissa(radius) ulps: both neighbours of r2 are reachable
    only for radii with a mantissa just above sqrt(2) whose square rounds by little.  So the radius used is the first
    f32 at or above `radius` for which every case is reached -> (pos_vis, {(geometry, kind): (i, j)}, radius used).
    Callers assert that every case was constructed."""
    r0 = np.array([np.float32(radius)]).view(np.int32)[0]
    rs = (r0 + np.arange(1 << 20, dtype=np.int32)).view(np.float32)
    up = (rs.view(np.int32) + 1).view(np.float32)
    dn = (rs.view(np.int32) - 1).view(np.float32)
    r2 = (rs * rs).astype(np.float32)
    ok = ((up * up).astype(np.float32).view(np.int32) == r2.view(np.int32) + 1) & \
         ((dn * dn).astype(np.float32).view(np.int32) == r2.view(np.int32) - 1)
    best = None
    for r in rs[ok][:64]:
        pos, where = _edge_cloud_at(float(r))
        if best is None or len(where) > len(best[1]):
            best = (pos, where, float(r))
        if len(where) == 3 * len(EDGE_KINDS):
            break
    return best


# ---- the grid's cell / bucket functions (select.cu), restated ---------------------------------------------------------

HX, HY, HZ = 0x9E3779B97F4A7C15, 0xC2B2AE3D27D4EB4F, 0x165667B19E3779F9
M64 = (1 << 64) - 1


def num_buckets(n: int) -> int:
    b = 1 << 10
    while b < n and b < (1 << 24):
        b <<= 1
    return b


def cell_of(p, radius: float):
    return tuple(_cell(float(x), radius) for x in p[:3])


def bucket_of(c, n_buckets: int) -> int:
    h = (c[0] * HX + c[1] * HY + c[2] * HZ) & M64
    h ^= h >> 29
    h = (h * 0xBF58476D1CE4E5B9) & M64
    h ^= h >> 32
    return h & (n_buckets - 1)


def neighbour_buckets(c, n_buckets: int):
    return [bucket_of((c[0] - 1 + k % 3, c[1] - 1 + k // 3 % 3, c[2] - 1 + k // 9), n_buckets) for k in range(27)]


def repeated_bucket_cloud(radius: float = 1.0, n: int = 1000, seed: int = 3):
    """A cloud of n <= 1024 gaussians (1024 buckets) in which the 27-cell scan of some gaussians meets one bucket twice:
      - `self`: a lone gaussian whose own cell shares its bucket with a neighbour cell (count 1; 2 if double-counted);
      - `pair`: a gaussian with one neighbour within radius, in a cell whose bucket another of the 27 cells shares
        (count 2; 3 if double-counted).
    Selecting with threshold 2 (self) and 3 (pair) tells a deduplicated scan from one that is not.
    -> (pos_vis, {"self": i, "pair": (i, j)})."""
    nb = num_buckets(n)
    assert nb == 1024
    cell = float(np.float32(radius)) * (1.0 + 1.0 / 1024.0)
    found = {}
    rng = range(-12, 12)
    for cx in rng:
        for cy in rng:
            for cz in rng:
                c = (cx, cy, cz)
                nbk = neighbour_buckets(c, nb)
                if "self" not in found and nbk.count(nbk[13]) > 1:
                    found["self"] = c
                dup = [k for k in range(27) if k != 13 and nbk.count(nbk[k]) > 1 and nbk.count(nbk[13]) == 1]
                far = "self" in found and max(abs(a - b) for a, b in zip(c, found["self"])) >= 4
                if "pair" not in found and dup and far:
                    found["pair"] = (c, dup[0])
                if len(found) == 2:
                    break
            if len(found) == 2:
                break
        if len(found) == 2:
            break
    assert len(found) == 2, "no repeated bucket among the 27 cells found in the search box"
    pts = []
    c = found["self"]
    pts.append([(c[0] + 0.5) * cell, (c[1] + 0.5) * cell, (c[2] + 0.5) * cell])
    c, k = found["pair"]
    pi =[(c[0] + 0.95) * cell if k % 3 == 2 else (c[0] + 0.05) * cell if k % 3 == 0 else (c[0] + 0.5) * cell,
          (c[1] + 0.95) * cell if k // 3 % 3 == 2 else (c[1] + 0.05) * cell if k // 3 % 3 == 0 else (c[1] + 0.5) * cell,
          (c[2] + 0.95) * cell if k // 9 == 2 else (c[2] + 0.05) * cell if k // 9 == 0 else (c[2] + 0.5) * cell]
    # j: just across the shared faces, in neighbour cell k, within 0.2 of i
    step = [(k % 3 - 1) * 0.1 * cell, (k // 3 % 3 - 1) * 0.1 * cell, (k // 9 - 1) * 0.1 * cell]
    pj = [pi[0] + step[0], pi[1] + step[1], pi[2] + step[2]]
    pts += [pi, pj]
    # filler far away (x > 1000): alone, in cells the two cases do not scan
    rs = np.random.default_rng(seed)
    fill = rs.uniform(0, 1, (n - 3, 3)) * [4000.0, 4000.0, 4000.0] + [1000.0, -2000.0, -2000.0]
    xyz = np.concatenate([np.array(pts), fill]).astype(np.float32)
    p = pos_cloud(xyz)
    return p, {"self": 0, "pair": (1, 2), "cells": found}
