"""The host halves of subset / download / save_selection, on the CPU: PlanarGaussian3d.from_f16 against pack_f16 on every
half pattern, the reach of tests/subset_cases.py over the selection predicate's classes, and the host side of
save_selection (subset -> writer -> reader)."""
import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
import subset_cases as S
from bevy_gaussian_splatting_b200.gaussian import compute_aabb


def all_halves_packed():
    """Every 16-bit pattern once in each half-word slot of the sh words and of the four second-plane words."""
    h = np.arange(65536, dtype=np.uint32)
    n = 65536 // 8                                   # (the second plane's 8 halves per gaussian take each pattern once)
    sh_h = np.resize(h, n * 48).reshape(n, 48)
    rs_h = np.resize(np.roll(h, 12345), n * 8).reshape(n, 8)
    sh = (sh_h[:, 1::2] << 16) | sh_h[:, 0::2]
    rso = np.stack([(rs_h[:, 2 * k] << 16) | rs_h[:, 2 * k + 1] for k in range(4)], axis=1)
    pos = np.arange(n * 4, dtype=np.float32).reshape(n, 4)
    return pos, sh.astype(np.uint32), rso.astype(np.uint32), sh_h, rs_h


def is_nan_half(bits):
    return ((bits & 0x7C00) == 0x7C00) & ((bits & 0x03FF) != 0)


def test_from_f16_inverts_pack_f16_on_every_half():
    pos, sh, rso, sh_h, rs_h = all_halves_packed()
    c = B.PlanarGaussian3d.from_f16(pos, sh, rso)
    assert c.position_visibility.tobytes() == pos.tobytes()
    sh2, rso2 = c.pack_f16()
    got_sh = np.stack([sh2 & 0xFFFF, sh2 >> 16], axis=2).reshape(len(sh2), 48)
    got_rs = np.stack([rso2 >> 16, rso2 & 0xFFFF], axis=2).reshape(len(rso2), 8)
    for want, got, f32 in ((sh_h, got_sh, c.spherical_harmonic),
                           (rs_h, got_rs, np.concatenate([c.rotation, c.scale_opacity], axis=1))):
        nan = is_nan_half(want)
        assert nan.sum() > 0 and (~nan).sum() > 60000
        assert np.array_equal(got[~nan], want[~nan])
        assert np.isnan(f32[nan]).all() and not np.isnan(f32[~nan]).any()
    # every pattern was reached in the sh slots and in the second-plane slots
    assert len(np.unique(sh_h)) == 65536 and len(np.unique(rs_h)) == 65536


def test_from_f16_slot_order():
    c = B.random_gaussians_3d_seeded(257, 3)
    r = c.rounded_to_f16()
    d = B.PlanarGaussian3d.from_f16(c.position_visibility, *c.pack_f16())
    for a, b in ((d.spherical_harmonic, r.spherical_harmonic), (d.rotation, r.rotation), (d.scale_opacity, r.scale_opacity)):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    cov = c.precomputed_covariance()
    dc = B.PlanarGaussian3d.from_f16(c.position_visibility, *cov.pack_f16())
    rc = cov.rounded_to_f16()
    assert np.array_equal(dc.rotation, rc.rotation) and np.array_equal(dc.scale_opacity, rc.scale_opacity)


def test_compute_aabb_function_matches_the_method():
    c = B.random_gaussians_3d_seeded(1000, 4)
    lo, hi = c.compute_aabb()
    lo2, hi2 = compute_aabb(c.position_visibility)
    assert np.array_equal(lo, lo2) and np.array_equal(hi, hi2)


def test_cases_reach_every_class():
    cases = S.cases()
    allv = np.concatenate([c["vis"] for c in cases])
    bits = set(allv.view(np.uint32).tolist())
    for name, (v, want) in S.SPECIALS.items():
        assert int(np.asarray(v, np.float32).view(np.uint32)) in bits, name
        assert bool(S.kept(np.array([v], np.float32))[0]) == want, name
    assert S.kept(np.array([0.5], np.float32))[0] and not S.kept(np.array([S.BELOW_HALF]))[0]
    names = [c["name"] for c in cases]
    assert any(c["vis"].size and S.kept(c["vis"]).all() for c in cases)
    assert any(not S.kept(c["vis"]).any() for c in cases)
    assert len(set(names)) == len(names)
    # kept / dropped transitions on each side of word (32) and CTA (256) boundaries, and sizes off both
    trans = set()
    for c in cases:
        k = S.kept(c["vis"]).astype(np.int8)
        trans.update((np.flatnonzero(np.diff(k)) + 1).tolist())
    for b in (32, 64, 256, 512, 1024, 2048, 4096):
        assert {b - 1, b, b + 1} & trans, b
    assert {255, 256, 257} <= trans | {256} and {31, 33} <= trans
    sizes = {len(c["vis"]) for c in cases}
    assert {1, 31, 32, 33, 255, 256, 257} <= sizes


@pytest.mark.parametrize("ext", [".gcloud", ".ply"])
def test_save_selection_host_half_round_trips(tmp_path, ext):
    c = B.random_gaussians_3d_seeded(500, 5)
    vis = S.cases()[0]["vis"][:500]
    c.position_visibility[:, 3] = vis
    idx = np.flatnonzero(S.kept(vis))
    assert 0 < len(idx) < 500
    sub = c.subset(idx)
    path = tmp_path / f"sel{ext}"
    if ext == ".gcloud":
        B.write_gcloud(path, sub)
    else:
        B.io.write_ply_3d(path, sub)
    back = B.load_cloud(path)
    if ext == ".gcloud":
        for a, b in ((back.position_visibility, sub.position_visibility), (back.spherical_harmonic, sub.spherical_harmonic),
                     (back.rotation, sub.rotation), (back.scale_opacity, sub.scale_opacity)):
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    else:
        k = len(idx)
        assert len(back) == k + 32 - k % 32             # the reader pads like ply.rs
        assert np.array_equal(back.position_visibility[:k, :3], sub.position_visibility[:, :3])
        assert np.array_equal(back.spherical_harmonic[:k, :3], sub.spherical_harmonic[:, :3])   # (f_rest: ply.rs's i / 16)
        assert np.allclose(back.scale_opacity[:k, 3], sub.scale_opacity[:, 3], rtol=1e-5, atol=1e-6)
        norm = sub.rotation / np.linalg.norm(sub.rotation, axis=1, keepdims=True)
        assert np.allclose(back.rotation[:k], norm, atol=1e-6)
