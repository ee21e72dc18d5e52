"""The transform oracle (transform_oracle/) against the rule in include/bgs.h, on the CPU: its SH rotation satisfies the
defining identity over the renderer's basis, is orthogonal and composes as the rotations do; its q_R is scipy's rotation
up to sign; it accepts and refuses exactly the matrices of tests/transform_cases.py; and its planes follow the rule's
position, scale, selection and untouched-lane clauses."""
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import transform_cases as TC
from transform_oracle import transform_oracle as TO

F = np.float32

# the renderer's basis constants (project.cu: c_shc)
SHC = np.array([0.28209479177387814, -0.4886025119029199, 0.4886025119029199, -0.4886025119029199,
                1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792,
                0.5462742152960396, -0.5900435899266435, 2.890611442640554, -0.4570457994644658,
                0.3731763325901154, -0.4570457994644658, 1.445305721320277, -0.5900435899266435])


def basis(d):
    """(..., 16): the renderer's SH basis (sh_basis) at unit directions d (..., 3), in f64."""
    x, y, z = d[..., 0], d[..., 1], d[..., 2]
    xx, yy, zz = x * x, y * y, z * z
    p = np.stack([np.ones_like(x), y, z, x, x * y, y * z, 2 * zz - xx - yy, x * z, xx - yy, y * (3 * xx - yy), x * y * z,
                  y * (4 * zz - xx - yy), z * (2 * zz - 3 * xx - 3 * yy), x * (4 * zz - xx - yy), z * (xx - yy),
                  x * (xx - 3 * yy)], -1)
    return p * SHC


def unit_dirs(rng, n):
    d = rng.normal(size=(n, 3))
    return d / np.linalg.norm(d, axis=1, keepdims=True)


ROTS = Rotation.random(6, random_state=7).as_matrix()


@pytest.mark.parametrize("l", [1, 2, 3])
def test_sh_rotation_satisfies_the_defining_identity(l):
    rng = np.random.default_rng(l)
    k0, m = l * l, 2 * l + 1
    for R in ROTS:
        E = TO.sh_matrix(R, l)
        d = unit_dirs(rng, 200)
        c = rng.normal(size=m)
        lhs = basis(d)[:, k0:k0 + m] @ (E @ c)          # the baked coefficients along d
        rhs = basis(d @ R)[:, k0:k0 + m] @ c             # the original's along R^T d (rows: (R^T d)^T = d^T R)
        assert np.abs(lhs - rhs).max() <= 1e-12


@pytest.mark.parametrize("l", [1, 2, 3])
def test_sh_rotation_is_orthogonal_and_composes(l):
    m = 2 * l + 1
    for a, b in zip(ROTS[:3], ROTS[3:]):
        Ea, Eb, Eab = TO.sh_matrix(a, l), TO.sh_matrix(b, l), TO.sh_matrix(a @ b, l)
        assert np.abs(Ea @ Ea.T - np.eye(m)).max() <= 1e-12
        # E = D^T composes as the rotations: E(R1 R2) = E(R1) E(R2) (so D(R1 R2) = D(R2) D(R1))
        assert np.abs(Eab - Ea @ Eb).max() <= 1e-12
    assert np.abs(TO.sh_matrix(np.eye(3), l) - np.eye(m)).max() <= 1e-12


@pytest.mark.parametrize("name", sorted(TC.ACCEPTED))
def test_quaternion_matches_scipy_up_to_sign(name):
    M = TC.ACCEPTED[name].astype(np.float64)
    q, s, _ = TO.params(TC.ACCEPTED[name])
    A = M[:3, :3]
    s_want = np.sqrt(np.sum(A * A) / 3.0)
    assert s == F(s_want)
    x, y, z, w = Rotation.from_matrix(A / s_want).as_quat()
    want = np.array([w, x, y, z])
    assert q[0] >= 0
    assert min(np.abs(q - want).max(), np.abs(q + want).max()) <= 1e-6, (q, want)


def test_validation_accepts_and_refuses_exactly_the_cases():
    for name, m in TC.ACCEPTED.items():
        assert TO.accepts(m), name
    for name, m in TC.REFUSED.items():
        assert not TO.accepts(m), name


@pytest.mark.parametrize("degree", TC.DEGREES)
@pytest.mark.parametrize("sel", [False, True])
def test_oracle_planes_follow_the_rule(degree, sel):
    c = TC.cloud(2000, degree, 3 + degree)
    planes = TC.planes_of(c, "f32")
    M = TC.ACCEPTED["general"]
    (pos, sh, rot, so), bound = TO.transform("f32", degree, planes, M, selected=sel)
    hit = TC.selected(planes[0][:, 3]) if sel else np.ones(len(pos), bool)
    want_pos = TC.mat4_point(M, planes[0])
    both = np.isnan(pos[hit, :3]) & np.isnan(want_pos[hit])
    assert np.all((pos[hit, :3].view(np.uint32) == want_pos[hit].view(np.uint32)) | both)
    assert np.array_equal(pos[:, 3].view(np.uint32), planes[0][:, 3].view(np.uint32))
    _, s, _ = TO.params(M)
    with np.errstate(all="ignore"):
        assert np.array_equal((s * planes[3][hit, :3]).view(np.uint32), so[hit, :3].view(np.uint32))
    assert np.array_equal(so[:, 3].view(np.uint32), planes[3][:, 3].view(np.uint32))
    # band 0 and padding untouched; untouched gaussians byte for byte
    k = 3 * (degree + 1) ** 2
    assert np.array_equal(sh[:, :3].view(np.uint32), planes[1][:, :3].view(np.uint32))
    assert np.array_equal(sh[:, k:].view(np.uint32), planes[1][:, k:].view(np.uint32))
    for a, b in zip((pos, sh, rot, so), planes):
        assert np.array_equal(a[~hit].view(np.uint32), b[~hit].view(np.uint32))
    assert np.all(bound[:, :3] == 0) and np.all(bound[:, k:] == 0)
    if degree:
        assert np.all(bound[hit, 3:k] > 0)


@pytest.mark.parametrize("layout", ["f16", "cov"])
def test_f16_opacity_and_zero_words_keep_their_bits(layout):
    c = TC.cloud(1000, 2, 5)
    planes = TC.planes_of(c, layout)
    (pos, shp, second), _ = TO.transform(layout, 2, planes, TC.ACCEPTED["general"])
    assert np.array_equal(second[:, 3] & 0xFFFF if layout == "f16" else second[:, 3], planes[2][:, 3] & 0xFFFF
                          if layout == "f16" else planes[2][:, 3])
    assert np.array_equal(shp[:, 14:], planes[1][:, 14:])   # degree 2: 27 halves + 1 pad half in 14 words


def test_identity_keeps_a_unit_cloud_close():
    c = TC.cloud(1000, 3, 9, special=False)
    planes = TC.planes_of(c, "f32")
    (pos, sh, rot, so), _ = TO.transform("f32", 3, planes, TC.ACCEPTED["identity"])
    assert np.array_equal(pos.view(np.uint32), planes[0].view(np.uint32))
    assert np.array_equal(rot.view(np.uint32), planes[2].view(np.uint32))
    assert np.abs(sh - planes[1]).max() <= 1e-6
