"""bgs_cloud_transform and bgs_cloud_bounds on the host side, without a GPU: the prototypes and mode constants, the NULL
refusals, the similarity_transform helper, and update_aabb's arithmetic (aabb_of_extent) against compute_aabb."""
import ctypes as C

import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
from bevy_gaussian_splatting_b200 import abi
from bevy_gaussian_splatting_b200.gaussian import aabb_of_extent, compute_aabb

F = np.float32


def test_prototypes_and_constants():
    names = {n: (r, a) for n, r, a in abi.SYMBOLS}
    assert names["bgs_cloud_transform"] == (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32])
    assert names["bgs_cloud_bounds"][1][2] is C.c_uint32
    assert (abi.BGS_TRANSFORM_ALL, abi.BGS_TRANSFORM_SELECTED) == (0, 1)


def test_null_arguments_are_refused():
    lib = abi.load()
    m = (C.c_float * 16)(*np.eye(4, dtype=F).reshape(-1))
    lo, hi, n = (C.c_float * 3)(), (C.c_float * 3)(), C.c_uint32()
    assert lib.bgs_cloud_transform(None, None, m, 0) == abi.BGS_EINVAL
    assert lib.bgs_cloud_transform(None, None, None, 1) == abi.BGS_EINVAL
    assert lib.bgs_cloud_bounds(None, None, 0, lo, hi, C.byref(n)) == abi.BGS_EINVAL
    assert lib.bgs_cloud_bounds(None, None, 0, None, None, None) == abi.BGS_EINVAL


def _apply(m, p):
    return (np.asarray(m, np.float64) @ np.append(np.asarray(p, np.float64), 1.0))[:3]


def test_similarity_transform_rotates_and_scales_about_the_pivot():
    rng = np.random.default_rng(1)
    for _ in range(20):
        q = rng.normal(size=4)
        t, pivot, s = rng.normal(size=3), rng.normal(size=3) * 5, float(rng.uniform(0.1, 3))
        m = B.similarity_transform(t, q, s, pivot)
        assert m.dtype == F and m.shape == (4, 4)
        assert np.array_equal(m[3], [0, 0, 0, 1])
        assert np.allclose(_apply(m, pivot), pivot + t, atol=1e-5)         # the pivot only moves by the translation
        A = m[:3, :3].astype(np.float64)
        assert np.allclose(A.T @ A, s * s * np.eye(3), atol=1e-5 * s * s)
        assert np.linalg.det(A) > 0
        qn = q / np.linalg.norm(q)
        from scipy.spatial.transform import Rotation
        R = Rotation.from_quat([qn[1], qn[2], qn[3], qn[0]]).as_matrix()
        assert np.allclose(A / s, R, atol=1e-6)
    assert np.array_equal(B.similarity_transform(), np.eye(4, dtype=F))


def test_similarity_transform_is_cloud_transform_convention():
    m = B.similarity_transform((1.0, 2.0, 3.0))
    u = B.GaussianSplattingPlugin.cloud_uniform(B.CloudSettings(), B.CloudTransform(m))
    assert list(u.transform)[12:15] == [1.0, 2.0, 3.0]     # column-major: the translation is the last column


@pytest.mark.parametrize("seed", range(5))
def test_aabb_of_extent_equals_compute_aabb(seed):
    rng = np.random.default_rng(seed)
    p = np.zeros((1000, 4), F)
    p[:, :3] = (rng.normal(size=(1000, 3)) * 10 ** rng.uniform(-3, 3)).astype(F)
    p[rng.integers(0, 1000, 5), 0] = -0.0
    want = compute_aabb(p)
    got = aabb_of_extent(p[:, :3].min(0), p[:, :3].max(0))
    for g, w in zip(got, want):
        assert np.array_equal(g.view(np.uint32), w.view(np.uint32))


def test_aabb_of_an_empty_extent_is_compute_aabbs_empty_box():
    want = compute_aabb(np.zeros((0, 4), F))
    got = aabb_of_extent(np.full(3, np.inf, F), np.full(3, -np.inf, F))
    for g, w in zip(got, want):
        assert np.array_equal(np.isnan(g), np.isnan(w)) and np.array_equal(g[~np.isnan(g)], w[~np.isnan(w)])
