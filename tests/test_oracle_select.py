"""SparseSelect's CPU oracle (select_oracle/): the brute force is the rule of include/bgs.h (checked against an
independent numpy float32 restatement), and the hashed grid -- the GPU kernel's cell and bucket functions, restated --
equals the brute force on every input class the GPU tests use, including knife-edge pairs and repeated buckets."""
import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
import select_cases as SC
from select_oracle import select_oracle as SO

THRESHOLDS = (0, 1, 2, 3, 64)


def both(pos, radius, thr):
    m_b, s_b = SO.select_sparse(pos, radius, thr)
    m_g, s_g = SO.select_sparse(pos, radius, thr, grid=True)
    assert s_b == int(m_b.sum()) and s_g == int(m_g.sum())
    assert np.array_equal(m_b, m_g), f"grid != brute force at {np.flatnonzero(m_b != m_g)[:8]} (radius {radius}, threshold {thr})"
    return m_b


@pytest.mark.parametrize("radius", [0.05, 0.5, 2.0, 7.0])
@pytest.mark.parametrize("thr", [1, 3, 64])
def test_brute_force_matches_numpy_restatement(radius, thr):
    for pos in (SC.uniform(1200, 1, 10.0), SC.with_duplicates(700, 2), SC.non_finite(500, 3)):
        m, _ = SO.select_sparse(pos, radius, thr)
        assert np.array_equal(m, SC.numpy_select(pos, radius, thr))


CLOUDS = {
    "uniform": lambda: SC.uniform(6000, 10),
    "clustered": lambda: SC.clustered(6000, 11),
    "duplicates": lambda: SC.with_duplicates(3000, 12),
    "non_finite": lambda: SC.non_finite(3000, 13),
    "large_coordinates": lambda: SC.large_coordinates(4000, 14),
}


@pytest.mark.parametrize("name", sorted(CLOUDS))
def test_grid_equals_brute_force(name):
    pos = CLOUDS[name]()
    radii = (1e-3, 0.05) if name == "large_coordinates" else (0.05, 0.3, 1.0, 2.5)
    for radius in radii + (0.0,):
        for thr in THRESHOLDS:
            m = both(pos, radius, thr)
            if thr == 0:
                assert not m.any()
            if radius == 0.0 and thr > 0:
                assert m.all()       # every count is 0
    if name == "non_finite":
        bad = ~np.isfinite(pos[:, :3]).all(1)
        assert bad.any()
        assert both(pos, 1.0, 1)[bad].all()    # count 0 < 1, whatever the radius
    if name == "large_coordinates":
        _, cells, _ = SO.buckets(pos, 1e-3)
        assert np.abs(cells).max() > 5e8      # cell coordinates near 1e9: the hash sees large keys
        m = both(pos, 1e-3, 2)
        assert 0 < m.sum() < len(m)           # duplicates are neighbours, lone points are not


def test_grid_equals_brute_force_on_ply_padding(tmp_path):
    """The .ply loader pads the cloud with default gaussians at the origin (ply.rs:127-129): many exact duplicates."""
    cloud = B.random_gaussians_3d_seeded(1000, 4)
    cloud.position_visibility[:, :3] *= np.float32(0.05)
    path = tmp_path / "c.ply"
    B.io.write_ply_3d(str(path), cloud)
    loaded = B.parse_ply_3d(str(path))
    assert len(loaded) == 1024 and np.all(loaded.position_visibility[1000:, :3] == 0)
    for thr in THRESHOLDS:
        m = both(loaded.position_visibility, 0.05, thr)
        if 0 < thr <= 24:
            assert not m[1000:].any()          # 24 padding gaussians at one point: never sparse below 25


def test_clamped_cells_merge_but_stay_exact():
    """A radius so small that cell coordinates saturate at +-2^40: cells merge, the decisions do not change."""
    pos = SC.uniform(2000, 21, 100.0)
    pos[::5, :3] = pos[1::5, :3]
    radius = 1e-12
    _, cells, _ = SO.buckets(pos, radius)
    assert np.abs(cells).max() == 2 ** 40
    for thr in (1, 2, 3):
        both(pos, radius, thr)


@pytest.mark.parametrize("nominal", [0.0884, 0.1768, 0.7072])
def test_knife_edge_pairs(nominal):
    pos, where, radius = SC.knife_edge_cloud(nominal)
    want = {(g, k) for g in ("axis", "diagonal", "boundary") for k in SC.EDGE_KINDS}
    assert set(where) == want, f"construction missed {sorted(want - set(where))}"
    t = SC._targets(radius)
    _, cells, _ = SO.buckets(pos, radius)
    for (geo, kind), (i, j) in where.items():
        assert SC.d2_f32(pos[i, :3], pos[j, :3]) == t[kind]
        if geo == "boundary":
            assert cells[i, 0] + 1 == cells[j, 0], "boundary pair does not straddle a cell boundary"
    m = both(pos, radius, 2)                      # selected iff alone (count 1 < 2)
    assert np.array_equal(m, SC.numpy_select(pos, radius, 2))
    for (geo, kind), (i, j) in where.items():
        # d2 == r2 and one ulp above: not neighbours; one ulp below: neighbours
        assert m[i] == m[j] == (kind != "below"), (geo, kind)


def test_repeated_buckets_are_scanned_once():
    pos, case = SC.repeated_bucket_cloud()
    b, cells, nb = SO.buckets(pos, 1.0)
    # the restated functions agree with the oracle's
    for i in (0, 1, 2, 10, 500):
        assert tuple(cells[i]) == SC.cell_of(pos[i], 1.0)
        assert b[i] == SC.bucket_of(SC.cell_of(pos[i], 1.0), nb)
    c_self = SC.cell_of(pos[case["self"]], 1.0)
    nbk = SC.neighbour_buckets(c_self, nb)
    assert nbk.count(nbk[13]) > 1                 # the lone gaussian's own bucket twice among its 27
    i, j = case["pair"]
    ci, cj = SC.cell_of(pos[i], 1.0), SC.cell_of(pos[j], 1.0)
    assert ci != cj and max(abs(a - b) for a, b in zip(ci, cj)) == 1
    nbk = SC.neighbour_buckets(ci, nb)
    assert nbk.count(SC.bucket_of(cj, nb)) > 1    # the neighbour's bucket twice among i's 27
    assert SC.d2_f32(pos[i, :3], pos[j, :3]) < np.float32(1.0)
    m2 = both(pos, 1.0, 2)
    assert m2[case["self"]] and not m2[i]
    m3 = both(pos, 1.0, 3)
    assert m3[i] and m3[j]


def test_bad_radius_is_refused():
    pos = SC.uniform(10, 0)
    for r in (float("nan"), float("inf"), -1.0):
        with pytest.raises(ValueError):
            SO.select_sparse(pos, r, 3)
