"""The point-in-mesh CPU oracle (select_oracle/): the brute force against an independent numpy float32 restatement of
raycast.rs:92-124, analytic answers, the literal quirks, and the grid restatement of libbgs's mesh_select.cu against
the brute force on every mesh case, knife-edge and sliver sets included."""
import numpy as np
import pytest

import mesh_cases as MC
from select_oracle import select_oracle as SO

F = np.float32


def numpy_hits(points: np.ndarray, v: np.ndarray, idx: np.ndarray) -> np.ndarray:
    """Hit count per point, raycast.rs:92-124 in numpy float32 (glam's scalar order, no contraction)."""
    o = points[:, None, :3].astype(F)
    v0, v1, v2 = (v[idx[:, k]][None].astype(F) for k in range(3))
    zero, one = F(0), F(1)
    eps = F(1e-6)
    with np.errstate(all="ignore"):
        e1, e2 = v1 - v0, v2 - v0
        d = (one, zero, zero)
        h = (d[1] * e2[..., 2] - e2[..., 1] * d[2], d[2] * e2[..., 0] - e2[..., 2] * d[0], d[0] * e2[..., 1] - e2[..., 0] * d[1])
        a = (e1[..., 0] * h[0] + e1[..., 1] * h[1]) + e1[..., 2] * h[2]
        ok = np.broadcast_to(~((a > -eps) & (a < eps)), o.shape[:1] + a.shape[1:]).copy()
        f = one / a
        s = o - v0
        u = f * ((s[..., 0] * h[0] + s[..., 1] * h[1]) + s[..., 2] * h[2])
        ok &= (u >= zero) & (u <= one)
        q = (s[..., 1] * e1[..., 2] - e1[..., 1] * s[..., 2], s[..., 2] * e1[..., 0] - e1[..., 2] * s[..., 0],
             s[..., 0] * e1[..., 1] - e1[..., 0] * s[..., 1])
        vv = f * ((d[0] * q[0] + d[1] * q[1]) + d[2] * q[2])
        ok &= ~((vv < zero) | (u + vv > one))
        t = f * ((e2[..., 0] * q[0] + e2[..., 1] * q[1]) + e2[..., 2] * q[2])
        ok &= t > eps
    return ok.sum(1)


def case_points(name, mesh):
    p = MC.scatter(mesh, 1500, hash(name) % 1000)
    if name in ("box", "inverted_box", "open_box", "non_finite", "far_triangles"):
        p = np.concatenate([p, MC.knife_points()])
    return p


@pytest.mark.parametrize("name", sorted(MC.MESHES))
def test_brute_force_equals_numpy_restatement(name):
    mesh = MC.MESHES[name]()
    p = case_points(name, mesh)[:400]
    m, n_in = SO.select_in_mesh(p, *mesh)
    want = numpy_hits(p, *mesh) % 2 == 1
    assert np.array_equal(m, want), np.flatnonzero(m != want)[:8]
    assert n_in == int(want.sum())


@pytest.mark.parametrize("name", sorted(MC.MESHES))
def test_grid_equals_brute_force(name):
    mesh = MC.MESHES[name]()
    p = case_points(name, mesh)
    m, n_in = SO.select_in_mesh(p, *mesh)
    g, g_in = SO.select_in_mesh(p, *mesh, grid=True)
    assert np.array_equal(m, g), np.flatnonzero(m != g)[:8]
    assert n_in == g_in


@pytest.mark.parametrize("offset", [0.0, 1e4])
def test_knife_points_grid_equals_brute_force(offset):
    v, i = MC.box()
    v = (v + F(offset)).astype(F)
    p = MC.knife_points(offset)
    M = np.eye(4, dtype=F)
    for mesh_from_cloud in (None, M):
        m, _ = SO.select_in_mesh(p, v, i, mesh_from_cloud)
        g, _ = SO.select_in_mesh(p, v, i, mesh_from_cloud, grid=True)
        assert np.array_equal(m, g)
        assert np.array_equal(m, numpy_hits(p, v, i) % 2 == 1)


def test_analytic_answers():
    # (off the faces' diagonals and the icosphere's edges: a ray through a shared edge counts both triangles)
    inside = MC.pts([(0.05, 0.13, -0.21), (0.5, -0.3, 0.2), (-0.7, 0.6, -0.45)])
    outside = MC.pts([(2.0, 0.0, 0.0), (-2.0, 0.1, 0.1), (0.0, 1.5, 0.0), (0.3, 0.2, -3.0)])
    for mesh in (MC.box(), MC.rotated_box(2), MC.icosphere(3), MC.inverted_box()):
        assert SO.select_in_mesh(inside[:1], *mesh)[0].all()
        assert not SO.select_in_mesh(outside, *mesh)[0].any()
    assert SO.select_in_mesh(inside, *MC.box())[0].all()
    tor = MC.torus(32, 16)
    ang = np.array([0.1, 2.0, 4.0])                        # off the mesh's seams
    tube = MC.pts(np.stack([np.full(3, 0.02), 1.01 * np.cos(ang), 1.01 * np.sin(ang)], 1))
    hole = MC.pts([(0.0, 0.0, 0.0), (-0.2, 0.1, 0.1)])
    assert SO.select_in_mesh(tube, *tor)[0].all()
    assert not SO.select_in_mesh(hole, *tor)[0].any()


def test_shared_edge_counts_both_triangles():
    # two triangles in the x = 0 plane sharing the edge y + z = 1
    v = np.array([(0, 0, 0), (0, 1, 0), (0, 0, 1), (0, 1, 1)], F)
    i = np.array([(0, 1, 2), (1, 3, 2)], np.uint32)
    p = MC.pts([(-1, 0.25, 0.25), (-1, 0.75, 0.75), (-1, 0.5, 0.5), (-1, 1.0, 0.0)])
    assert list(numpy_hits(p, v, i)) == [1, 1, 2, 2]       # on the shared edge / vertex: both triangles hit
    m, _ = SO.select_in_mesh(p, v, i)
    assert list(m) == [True, True, False, False]


def test_tiny_triangles_are_never_hit():
    v, i = MC.slivers()
    cls, _ = SO.mesh_boxes(v, i)
    a = np.array([1e-6], F)[0]
    # |a| one ulp below 1e-6 is rejected, at or above it survives
    assert list(cls[:6]) == [0, 2, 2, 2, 0, 2]             # the survivors are slivers: tested against every point
    assert cls[6] == 0 and cls[7] == 2
    # the tiny one: its whole interior misses
    p = MC.pts([(-1, 0.10002, 0.10002), (-1, 0.10001, 0.10003)])
    assert not SO.select_in_mesh(p, v[18:21], i[:1])[0].any()
    assert a == F(1e-6)


def test_non_finite_never_hits():
    v, i = MC.non_finite()
    bad = i[12:]
    pts = MC.scatter((v[:8], i[:12]), 2000, 7)
    assert (numpy_hits(pts, v, bad) == 0).all()
    assert not SO.select_in_mesh(pts, v, bad)[0].any()
    cls, _ = SO.mesh_boxes(v, bad)
    assert (cls == 0).all()                                # a is NaN or infinite for every one of them
    nf = MC.pts([(np.inf, 0, 0), (-np.inf, 0, 0), (0, np.inf, 0), (0, 0, -np.inf), (np.nan, 0, 0), (0, np.nan, 0)])
    assert (numpy_hits(nf, *MC.box()) == 0).all()
    assert not SO.select_in_mesh(nf, *MC.box())[0].any()


def test_grid_cases_reach_every_class_and_level():
    plan = SO.mesh_plan(*MC.coarsening())
    assert plan["level"] > 0                               # the pair budget forced coarsening
    assert plan["pairs"] <= (1 << 24) + 4 * plan["binned"]
    assert SO.mesh_plan(*MC.all_rejected()) == {"binned": 0, "global": 0, "ny": 0, "nz": 0, "level": -1, "pairs": 0}
    assert SO.mesh_plan(*MC.far_triangles())["global"] == 2
    assert SO.mesh_plan(*MC.slivers())["global"] >= 1
    big = SO.mesh_plan(*MC.big_and_small())
    assert big["level"] == 0 and big["ny"] * big["nz"] > 1000


def test_accepted_points_lie_in_the_widened_box():
    """Every point the f32 test accepts lies inside the triangle's slack-widened box (the grid's claim), for triangles
    at offsets up to 1e4 and points a few ulps around their vertices."""
    rng = np.random.default_rng(11)
    for k in range(200):
        c = rng.uniform(-1e4, 1e4, 3)
        t = (c + rng.normal(0, 1.0, (3, 3))).astype(F)
        v, i = t, np.array([[0, 1, 2]], np.uint32)
        cls, box = SO.mesh_boxes(v, i)
        if cls[0] != 1:
            continue
        p = []
        for vert in t:
            for dy in range(-3, 4):
                for dz in range(-3, 4):
                    y, z = vert[1], vert[2]
                    for _ in range(abs(dy)):
                        y = np.nextafter(y, F(np.inf) if dy > 0 else F(-np.inf))
                    for _ in range(abs(dz)):
                        z = np.nextafter(z, F(np.inf) if dz > 0 else F(-np.inf))
                    p.append((vert[0] - F(5), y, z))
        p = MC.pts(p)
        m, _ = SO.select_in_mesh(p, v, i)
        assert m.any()
        g, _ = SO.select_in_mesh(p, v, i, grid=True)
        assert np.array_equal(m, g)
        assert (p[m, 1] >= box[0, 0]).all() and (p[m, 1] <= box[0, 1]).all()
        assert (p[m, 2] >= box[0, 2]).all() and (p[m, 2] <= box[0, 3]).all()


def test_transform_and_bad_indices():
    v, i = MC.box()
    p = MC.scatter((v, i), 3000, 3)
    M = np.eye(4, dtype=np.float64)
    M[:3, :3] = MC.rotation(5) @ np.diag([1.5, 0.5, 2.0])
    M[:3, 3] = (0.3, -0.2, 0.1)
    M = M.astype(F)
    m, _ = SO.select_in_mesh(p, v, i, M)
    g, _ = SO.select_in_mesh(p, v, i, M, grid=True)
    assert np.array_equal(m, g)
    q = np.ascontiguousarray(np.concatenate([((M[:3, :3].astype(F) @ p[:, :3].T).T), np.ones((len(p), 1), F)], 1))
    assert 0 < m.sum() < len(p)
    with pytest.raises(ValueError):
        SO.select_in_mesh(p, v, np.array([[0, 1, 8]], np.uint32))
    assert q.shape == p.shape
