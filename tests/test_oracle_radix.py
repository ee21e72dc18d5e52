"""Oracle pinned against the reference's own pure tests for the sort key / pass plan.

Each test restates one test of the reference's tests/radix.rs (file:line in the docstring) against
the ORACLE's key formula and pass plan, plus the ABI-side mirror `ShaderDefines`.
"""
import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B

IDENT = np.eye(4, dtype=np.float32)


def _view_at(cam, w=64, h=64):
    return B.perspective_view(cam, (cam[0], cam[1], cam[2] + 1.0), w, h)   # looking +Z at the test points


def _keys(oracle, positions, cam, bits):
    pos = np.array([[*p, 1.0] for p in positions], np.float32)
    view = _view_at(cam)
    u = B.GaussianSplattingPlugin.cloud_uniform(B.CloudSettings())
    return oracle.keygen(pos, view.to_abi(), u, bits)


def _dist2(p, c):
    d = np.float32(p) - np.float32(c)
    return np.float32(np.float32(d[0] * d[0] + d[1] * d[1]) + d[2] * d[2])


def test_radix_depth_key_formula(oracle):
    """tests/radix.rs:96-106: key = (0xFFFFFFFF - bits(dist2)) >> shift for in-frustum points."""
    pts = [(-0.02, 0.0, 1.0), (0.02, 0.0, 1.0), (0.3, -0.2, 7.5)]
    cam = (-0.01, 0.0, 0.0)
    for bits in (16, 24, 32):
        shift = 32 - bits
        got = _keys(oracle, pts, cam, bits)
        for p, k in zip(pts, got):
            want = (0xFFFFFFFF - int(np.float32(_dist2(p, cam)).view(np.uint32))) >> shift
            assert int(k) == want


def test_radix_depth_key_preserves_close_order_during_camera_motion(oracle):
    """tests/radix.rs:10-39: ascending key order stays back-to-front at 24/32 bits."""
    positions = [(-0.02, 0.0, 1.0), (0.02, 0.0, 1.0)]
    for bits in (24, 32):
        for cam in [(-0.01, 0.0, 0.0), (0.01, 0.0, 0.0)]:
            keys = _keys(oracle, positions, cam, bits)
            order = oracle.stable_sort(keys)
            d = [float(_dist2(positions[i], cam)) for i in order]
            assert all(d[i] >= d[i + 1] for i in range(len(d) - 1)), (bits, cam, keys)


def test_radix_depth_bit_settings_select_expected_pass_count_and_shift(oracle):
    """tests/radix.rs:42-62: (places, shift, initial parity) = (2,16,0) / (3,8,1) / (4,0,0)."""
    cases = [(16, 2, 16, 0), (24, 3, 8, 1), (32, 4, 0, 0)]
    for bits, places, shift, parity in cases:
        assert oracle.pass_plan(bits) == (places, shift, parity)
        d = B.ShaderDefines.for_radix_depth_bits(B.RadixSortDepthBits(bits))
        assert (d.radix_digit_places, d.radix_key_shift, d.radix_initial_parity()) == (places, shift, parity)


def test_radix_initial_parity_finishes_in_sorted_entries_buffer(oracle):
    """tests/radix.rs:65-79: the last pass writes sorted_entries; the oracle's literal ping-pong
    returns non-zero if it would not."""
    rng = np.random.default_rng(0)
    keys = rng.integers(0, 2**32, 5000, dtype=np.uint64).astype(np.uint32)
    for bits in (16, 24, 32):
        places, shift, parity = oracle.pass_plan(bits)
        assert (parity + places - 1) % 2 == 1
        sk, si = oracle.radix_sort(keys >> shift, bits)   # asserts rc == 0 inside
        assert np.all(sk[:-1] <= sk[1:])


def test_radix_16_bit_depth_key_can_collapse_close_depths(oracle):
    """tests/radix.rs:82-94."""
    keys = _keys(oracle, [(-0.02, 0.0, 1.0), (0.02, 0.0, 1.0)], (-0.01, 0.0, 0.0), 16)
    assert keys[0] == keys[1]


@pytest.mark.parametrize("bits", [16, 24, 32])
def test_lsd_radix_equals_stable_sort(oracle, bits):
    """a3: the literal LSD pass structure == std::stable_sort ascending (ties keep index order)."""
    rng = np.random.default_rng(bits)
    n = 20011
    keys = (rng.integers(0, 2**32, n, dtype=np.uint64).astype(np.uint32)) >> (32 - bits)
    keys[rng.integers(0, n, n // 3)] = keys[0]                # many ties
    keys[rng.integers(0, n, n // 5)] = 0xFFFFFFFF >> (32 - bits)   # "culled"
    sk, si = oracle.radix_sort(keys, bits)
    assert np.array_equal(si, oracle.stable_sort(keys))
    assert np.array_equal(sk, keys[si])
    assert np.array_equal(si, np.argsort(keys, kind="stable").astype(np.uint32))


def test_culled_entries_key_all_ones_and_sort_last(oracle):
    """radix.wgsl:86-101: out-of-frustum -> 0xFFFFFFFF (then shifted); they end up last, index order."""
    cloud = B.random_gaussians_3d_seeded(4000, 3)
    view = B.headless_view(128, 128)
    u = B.GaussianSplattingPlugin.cloud_uniform(B.CloudSettings())
    for bits in (16, 24, 32):
        keys = oracle.keygen(cloud.position_visibility, view.to_abi(), u, bits)
        culled = 0xFFFFFFFF >> (32 - bits)
        nv = int((keys != culled).sum())
        assert 0 < nv < len(keys)
        sk, si = oracle.radix_sort(keys, bits)
        assert np.all(sk[nv:] == culled) and np.all(sk[:nv] != culled)
        assert np.all(np.diff(si[nv:].astype(np.int64)) > 0)


def test_keygen_empty_and_degenerate(oracle):
    view = B.headless_view(64, 64)
    u = B.GaussianSplattingPlugin.cloud_uniform(B.CloudSettings())
    assert len(oracle.keygen(np.zeros((0, 4), np.float32), view.to_abi(), u, 32)) == 0
    # a gaussian exactly at the camera: w = 0 -> ndc = 0/1e-9 -> z test fails -> culled
    pos = np.array([[0.0, 1.5, 5.0, 1.0], [np.nan, 0, 0, 1.0], [0.0, 1.5, -1e30, 1.0]], np.float32)
    keys = oracle.keygen(pos, view.to_abi(), u, 32)
    assert keys[0] == 0xFFFFFFFF and keys[1] == 0xFFFFFFFF
