"""Triangle meshes and point sets for the point-in-mesh selection tests, built in-process from seeds.

A mesh is (vertices (nv, 3) float32, indices (nt, 3) uint32).  Points are (n, 4) float32 pos_vis rows (visibility 1).
"""
import numpy as np

F = np.float32


def box(lo=(-1.0, -1.0, -1.0), hi=(1.0, 1.0, 1.0)):
    """Axis-aligned box, 12 outward-wound triangles."""
    lo, hi = np.asarray(lo, F), np.asarray(hi, F)
    v = np.array([[x, y, z] for x in (lo[0], hi[0]) for y in (lo[1], hi[1]) for z in (lo[2], hi[2])], F)
    # vertex k = 4 bx + 2 by + bz
    quads = [(0, 1, 3, 2), (4, 6, 7, 5), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3)]
    idx = []
    for a, b, c, d in quads:
        idx += [(a, b, c), (a, c, d)]
    return v, np.array(idx, np.uint32)


def rotation(seed: int) -> np.ndarray:
    q = np.random.default_rng(seed).normal(size=4)
    w, x, y, z = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def rotated_box(seed: int = 1):
    v, i = box((-1.0, -0.5, -0.75), (1.0, 0.5, 0.75))
    return (v.astype(np.float64) @ rotation(seed).T).astype(F), i


def icosphere(subdiv: int = 3, radius: float = 1.0):
    """20 * 4^subdiv triangles (subdiv 5: 20480)."""
    t = (1.0 + 5 ** 0.5) / 2.0
    v = [(-1, t, 0), (1, t, 0), (-1, -t, 0), (1, -t, 0), (0, -1, t), (0, 1, t), (0, -1, -t), (0, 1, -t),
         (t, 0, -1), (t, 0, 1), (-t, 0, -1), (-t, 0, 1)]
    v = [np.array(p, np.float64) / np.linalg.norm(p) for p in v]
    f = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2), (10, 7, 6),
         (7, 1, 8), (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11), (6, 2, 10), (8, 6, 7),
         (9, 8, 1)]
    for _ in range(subdiv):
        cache, nf = {}, []

        def mid(a, b):
            k = (min(a, b), max(a, b))
            if k not in cache:
                m = v[a] + v[b]
                v.append(m / np.linalg.norm(m))
                cache[k] = len(v) - 1
            return cache[k]
        for a, b, c in f:
            ab, bc, ca = mid(a, b), mid(b, c), mid(c, a)
            nf += [(a, ab, ca), (b, bc, ab), (c, ca, bc), (ab, bc, ca)]
        f = nf
    return (np.array(v) * radius).astype(F), np.array(f, np.uint32)


def torus(n_major: int = 48, n_minor: int = 24, R: float = 1.0, r: float = 0.35):
    """2 * n_major * n_minor triangles, genus 1, the hole along x (so +x rays cross it)."""
    a = np.arange(n_major) * 2 * np.pi / n_major
    b = np.arange(n_minor) * 2 * np.pi / n_minor
    A, Bm = np.meshgrid(a, b, indexing="ij")
    # ring in the yz plane: the +x ray from a point in the hole misses the tube
    x = r * np.sin(Bm)
    y = (R + r * np.cos(Bm)) * np.cos(A)
    z = (R + r * np.cos(Bm)) * np.sin(A)
    v = np.stack([x, y, z], -1).reshape(-1, 3).astype(F)
    idx = []
    for i in range(n_major):
        for j in range(n_minor):
            p = i * n_minor + j
            q = ((i + 1) % n_major) * n_minor + j
            p1 = i * n_minor + (j + 1) % n_minor
            q1 = ((i + 1) % n_major) * n_minor + (j + 1) % n_minor
            idx += [(p, q, q1), (p, q1, p1)]
    return v, np.array(idx, np.uint32)


def open_box():
    v, i = box()
    return v, i[2:]                       # the -x face missing


def inverted_box():
    v, i = box()
    return v, i[:, ::-1].copy()


def slivers():
    """Triangles whose `a` is one ulp either side of 1e-6 (and exactly at it), in the yz plane at x = 0."""
    eps = F(1e-6)
    tris = []
    for a in (np.nextafter(eps, F(0)), eps, np.nextafter(eps, F(1)), F(-eps), np.nextafter(F(-eps), F(0)),
              np.nextafter(F(-eps), F(-1))):
        # e1 = (0, 0, 1), e2 = (0, a, 0) -> h = (0, 0, a), a = e1 . h = a (exact)
        tris.append([(0.0, 0.0, 0.0), (0.0, 0.0, 1.0), (0.0, float(a), 0.0)])
    # tiny triangle (yz extent 1e-4: |a| ~ 5e-9 < eps, never hit) and a long thin sliver (kappa > 2^16: global)
    tris.append([(0.0, 0.1, 0.1), (0.0, 0.1001, 0.1), (0.0, 0.1, 0.1001)])
    tris.append([(0.0, -3.0, -2.0), (0.0, 3.0, 2.0), (0.0, 3.0, 2.00001)])
    v = np.array(tris, F).reshape(-1, 3)
    return v, np.arange(len(v), dtype=np.uint32).reshape(-1, 3)


def non_finite():
    """A box plus triangles with inf / NaN vertex coordinates (x, y or z; one or several vertices)."""
    v, i = box()
    extra = []
    for bad in (np.inf, -np.inf, np.nan):
        for k in range(3):
            for vert in range(3):
                t = np.array([(0.5, -0.5, -0.5), (0.5, 0.5, -0.5), (0.5, -0.5, 0.5)], np.float64)
                t[vert, k] = bad
                extra.append(t)
    ev = np.array(extra, F).reshape(-1, 3)
    ei = (np.arange(len(ev), dtype=np.uint32) + len(v)).reshape(-1, 3)
    return np.concatenate([v, ev]), np.concatenate([i, ei])


def big_and_small(seed: int = 3, n_small: int = 2000):
    """One triangle covering the whole grid among many small ones."""
    rng = np.random.default_rng(seed)
    c = rng.uniform(-1, 1, (n_small, 1, 3))
    t = c + rng.normal(0, 0.02, (n_small, 3, 3))
    big = np.array([[[0.0, -100.0, -100.0], [0.0, 100.0, -100.0], [0.0, 0.0, 100.0]]])
    v = np.concatenate([t, big]).astype(F).reshape(-1, 3)
    return v, np.arange(len(v), dtype=np.uint32).reshape(-1, 3)


def all_rejected(n: int = 500, seed: int = 4):
    """Every triangle parallel to the ray (zero yz area) or below the eps: no survivor."""
    rng = np.random.default_rng(seed)
    t = rng.uniform(-1, 1, (n, 3, 3))
    t[: n // 2, :, 1] = t[: n // 2, :1, 1]                # constant y: a == 0
    t[n // 2:, :, 1:] = t[n // 2:, :1, 1:] + rng.uniform(-1e-4, 1e-4, (n - n // 2, 3, 2))   # tiny yz extent
    v = t.astype(F).reshape(-1, 3)
    return v, np.arange(len(v), dtype=np.uint32).reshape(-1, 3)


def coarsening(n: int = 6000, seed: int = 5):
    """Many large overlapping triangles: level 0's pairs exceed the budget, the grid coarsens."""
    rng = np.random.default_rng(seed)
    t = rng.uniform(-1, 1, (n, 3, 3))
    t[:, :, 1:] *= 1.0
    t[:, 0, 1:] = (-1.0, -1.0)
    t[:, 1, 1:] = (1.0, -1.0) + rng.uniform(-0.05, 0.0, (n, 2))
    t[:, 2, 1:] = (0.0, 1.0) + rng.uniform(-0.05, 0.05, (n, 2))
    v = t.astype(F).reshape(-1, 3)
    return v, np.arange(len(v), dtype=np.uint32).reshape(-1, 3)


def far_triangles():
    """A box plus triangles with coordinates at or beyond 2^62 (tested against every point)."""
    v, i = box()
    t = np.array([[(0.5, -2.0, -2.0), (0.5, 2.0, -2.0), (2.0 ** 63, 0.0, 2.0)],
                  [(3.0, -5e18, -5e18), (3.0, 5e18, -5e18), (3.0, 0.0, 5e18)]], F).reshape(-1, 3)
    return np.concatenate([v, t]), np.concatenate([i, (np.arange(6, dtype=np.uint32) + len(v)).reshape(-1, 3)])


MESHES = {
    "box": box,
    "rotated_box": rotated_box,
    "icosphere": lambda: icosphere(3),
    "torus": lambda: torus(32, 16),
    "open_box": open_box,
    "inverted_box": inverted_box,
    "slivers": slivers,
    "non_finite": non_finite,
    "big_and_small": big_and_small,
    "all_rejected": all_rejected,
    "coarsening": coarsening,
    "far_triangles": far_triangles,
}


def pts(xyz) -> np.ndarray:
    xyz = np.asarray(xyz, F).reshape(-1, 3)
    return np.concatenate([xyz, np.ones((len(xyz), 1), F)], 1)


def scatter(mesh, n: int, seed: int) -> np.ndarray:
    """Points spread over the mesh's finite bounds (+25 %), plus points on and next to its vertices (+-1..4 ulps in y, z)."""
    rng = np.random.default_rng(seed)
    v = mesh[0][np.isfinite(mesh[0]).all(1) & (np.abs(mesh[0]) < 1e6).all(1)]
    if len(v) == 0:
        v = np.zeros((1, 3), F)
    lo, hi = v.min(0), v.max(0)
    c, e = (lo + hi) / 2, np.maximum((hi - lo) * 0.625, 1e-3)
    p = rng.uniform(c - e, c + e, (n, 3)).astype(F)
    k = min(n // 4, len(v) * 8)
    if k:
        base = v[rng.integers(0, len(v), k)].copy()
        base[:, 0] -= rng.uniform(0.01, 0.5, k).astype(F)
        for ax in (1, 2):
            steps = rng.integers(-4, 5, k)
            for j in range(k):
                for _ in range(abs(int(steps[j]))):
                    base[j, ax] = np.nextafter(base[j, ax], F(np.inf) if steps[j] > 0 else F(-np.inf))
        p[:k] = base
    return pts(p)


def knife_points(offset: float = 0.0):
    """Points of the unit box (offset along every axis) exactly on shared edges and vertices (in yz projection),
    one ulp either side of an edge in y and in z, and on the t = eps boundary of the -x... +x faces."""
    o = F(offset)
    lo, hi = F(-1) + o, F(1) + o
    up, dn = lambda a: np.nextafter(F(a), F(np.inf)), lambda a: np.nextafter(F(a), F(-np.inf))
    x0 = F(o - F(2))
    rows = []
    for y in (lo, hi, o, dn(lo), up(lo), dn(hi), up(hi)):
        for z in (lo, hi, o, dn(lo), up(lo), dn(hi), up(hi)):
            rows.append((x0, y, z))
            rows.append((o, y, z))
    # t = eps: the +x face at x = hi; t = hi - x (f = 1/a, |e2| = 2): points at x = hi - eps and one ulp either side
    for x in (F(hi - F(1e-6)), dn(F(hi - F(1e-6))), up(F(hi - F(1e-6))), hi, dn(hi)):
        rows.append((x, o + F(0.25), o + F(0.3)))
    # the shared diagonal of the +x face's two triangles (0, 1, 3) / (0, 3, 2) in box(): y == z
    for s in (F(-0.5), F(0.0), F(0.5), F(0.123)):
        rows.append((x0, o + s, o + s))
    return pts(rows)
