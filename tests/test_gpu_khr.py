"""bgs_cloud_upload_khr on the GPU: the decoded planes bit for bit against the CPU restatement of the reference's readers
(khr_oracle) for every accepted accessor combination, layout and size; every refusal, after which the context still
renders; scene frames against clouds uploaded from the oracle's decode; camera views; and the writer's round trip."""
import ctypes as C
import os
import warnings

import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
from bevy_gaussian_splatting_b200 import abi
from bevy_gaussian_splatting_b200.camera import look_at_rh
from khr_cases import A_COLOR, A_OP, A_POS, A_ROT, A_SCALE, COMBOS, GOLDEN, GltfBuilder, primitive_arrays, scene_of, sh_name
from khr_oracle import khr_oracle as K

pytestmark = pytest.mark.gpu

ROUNDED_TOL = 4e-3
CASE = {c[0]: c for c in COMBOS}


@pytest.fixture(scope="module")
def plugin():
    p = B.GaussianSplattingPlugin(0)
    yield p
    p.destroy()


def _upload(p, prim, f16):
    h, zq, d = C.c_void_p(), C.c_uint32(), prim.to_abi()
    rc = p._lib.bgs_cloud_upload_khr(p._ctx, C.byref(d), int(f16), C.byref(zq), C.byref(h))
    return rc, h, int(zq.value)


def _assert_parity(p, prim):
    want, zero = K.decode(prim)
    sh_p, rso = want.pack_f16()
    for f16 in (False, True):
        rc, h, zq = _upload(p, prim, f16)
        assert rc == abi.BGS_OK, p._lib.bgs_last_error(p._ctx)
        handle = B.PlanarGaussian3dHandle._adopt(p, h, prim.n, f16, False, aabb=want.compute_aabb())
        try:
            assert zq == zero and handle.sh_degree == want.sh_degree
            got = p.download_planes(handle)
            ref = (want.position_visibility, sh_p, rso) if f16 else \
                (want.position_visibility, want.spherical_harmonic, want.rotation, want.scale_opacity)
            for g, r in zip(got, ref):
                np.testing.assert_array_equal(g.view(np.uint32), np.ascontiguousarray(r).view(np.uint32))
        finally:
            handle.destroy()
    return zero


@pytest.mark.parametrize("n", [1, 31, 32, 33, 257])
@pytest.mark.parametrize("layout", ["packed", "interleaved", "offset"])
@pytest.mark.parametrize("combo", COMBOS, ids=[c[0] for c in COMBOS])
def test_decode_parity(plugin, combo, layout, n):
    kw = {"packed": {}, "interleaved": {"interleave": True}, "offset": {"offset": 12, "interleave": n % 2 == 1}}[layout]
    scene = scene_of(primitive_arrays(combo, n, n * 7 + len(layout)), **kw)
    assert _assert_parity(plugin, scene.primitives[0]) >= len(range(0, n, 7))   # (every 7th rotation is zero)


@pytest.mark.parametrize("combo", [CASE[k] for k in ("rot_f32", "rot_i16n", "scale_int16", "color4_uint16n", "sh3")],
                         ids=lambda c: c[0])
def test_decode_parity_large(plugin, combo):
    n = (1 << 20) + 3
    arrays = primitive_arrays(combo, n, 11)
    if combo[0] == "rot_f32":   # the quantised arrangement: i8 rotation, i16 scale, u8 opacity, SH degree 3
        rng = np.random.default_rng(12)
        rot = rng.integers(-128, 128, (n, 4)).astype(np.int8)
        rot[::7] = 0
        arrays[A_ROT] = (rot, True)
        arrays[A_SCALE] = (rng.integers(-32768, 32768, (n, 3)).astype(np.int16), True)
        arrays[A_OP] = (rng.integers(0, 256, (n, 1)).astype(np.uint8), True)
        for k in range(16):
            arrays[sh_name(k)] = (rng.uniform(-1, 1, (n, 3)).astype(np.float32), False)
    assert _assert_parity(plugin, scene_of(arrays, interleave=combo[0] == "scale_int16").primitives[0]) > 0


# ---- refusals

def _small_cloud_frame(p):
    h = p.add_cloud(B.random_gaussians_3d_seeded(2000, 3))
    try:
        return p.render_view(h, B.CloudSettings(), B.perspective_view((0, 0, 40), (0, 0, 0), 96, 64)).copy()
    finally:
        h.destroy()


def _refusal(p, prim, match):
    rc, h, _ = _upload(p, prim, False)
    assert rc == abi.BGS_EINVAL and not h.value
    assert match in p._lib.bgs_last_error(p._ctx).decode()


@pytest.mark.parametrize("slot,row,value,match", [
    (A_POS, 3, np.nan, "POSITION"), (A_POS, 0, np.inf, "POSITION"), (A_ROT, 5, np.nan, "ROTATION"),
    (A_SCALE, 9, 100.0, "SCALE"), (A_OP, 2, 1.5, "OPACITY"), (A_OP, 40, -0.1, "OPACITY"), (A_OP, 63, np.nan, "OPACITY"),
    (sh_name(3), 7, np.nan, "SH"), (A_COLOR, 1, np.inf, "COLOR_0")])
def test_device_rules_refuse(plugin, slot, row, value, match):
    before = _small_cloud_frame(plugin)
    combo = CASE["color4_f32" if slot == A_COLOR else "sh3"]
    arrays = primitive_arrays(combo, 64, 5)
    v, norm = arrays[slot]
    v = v.copy()
    v[row, 0] = value
    arrays[slot] = (v, norm)
    _refusal(plugin, scene_of(arrays).primitives[0], match)
    with pytest.raises(ValueError):
        K.decode(scene_of(arrays).primitives[0])
    np.testing.assert_array_equal(_small_cloud_frame(plugin), before)


def test_descriptor_rules_refuse(plugin):
    before = _small_cloud_frame(plugin)
    scene = scene_of(primitive_arrays(CASE["sh3"], 16, 2))
    prim = scene.primitives[0]

    def edit(fn, match):
        d = prim.to_abi()
        fn(d)
        h = C.c_void_p()
        assert plugin._lib.bgs_cloud_upload_khr(plugin._ctx, C.byref(d), 0, None, C.byref(h)) == abi.BGS_EINVAL and not h.value
        assert match in plugin._lib.bgs_last_error(plugin._ctx).decode()

    edit(lambda d: setattr(d.position, "component_type", 5122), "POSITION")
    edit(lambda d: setattr(d.position, "components", 4), "POSITION")
    edit(lambda d: setattr(d.rotation, "normalized", 0) or setattr(d.rotation, "component_type", 5120), "ROTATION")
    edit(lambda d: setattr(d.rotation, "component_type", 5121), "ROTATION")
    edit(lambda d: setattr(d.scale, "component_type", 5121), "SCALE")
    edit(lambda d: setattr(d.opacity, "normalized", 0) or setattr(d.opacity, "component_type", 5121), "OPACITY")
    edit(lambda d: setattr(d.opacity, "components", 3), "OPACITY")
    edit(lambda d: setattr(d.sh[5], "component_type", 5121), "SH_DEGREE_2_COEF_1")
    edit(lambda d: setattr(d.sh[15], "data", None), "SH_DEGREE_3_COEF_6")
    edit(lambda d: setattr(d.scale, "data", None), "SCALE")
    edit(lambda d: setattr(d.position, "byte_stride", 8), "POSITION")
    edit(lambda d: setattr(d.rotation, "byte_stride", 18), "ROTATION")
    edit(lambda d: setattr(d, "n", 0), "n must be")
    edit(lambda d: setattr(d, "n", 1 << 30), "n must be")
    edit(lambda d: setattr(d, "sh_degree", 4), "sh_degree")
    color = scene_of(primitive_arrays(CASE["color4_uint8"], 16, 2)).primitives[0]
    d = color.to_abi()
    d.color_0.component_type = 5120
    h = C.c_void_p()
    assert plugin._lib.bgs_cloud_upload_khr(plugin._ctx, C.byref(d), 0, None, C.byref(h)) == abi.BGS_EINVAL
    assert "COLOR_0" in plugin._lib.bgs_last_error(plugin._ctx).decode()
    np.testing.assert_array_equal(_small_cloud_frame(plugin), before)


# ---- frames

def _oracle_entities(p, scene, f16):
    handles = [p.add_cloud(K.decode(prim)[0], f16=f16) for prim in scene.primitives]
    return handles, [(handles[b.primitive], b.settings, b.transform) for b in scene.bundles]


@pytest.mark.parametrize("fmt", ["rgba32f", "rgba16f", "rgba8_srgb"])
@pytest.mark.parametrize("f16", [False, True])
def test_fixture_frames_match_oracle_clouds(plugin, fmt, f16):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        scene = B.load_scene(os.path.join(GOLDEN, "khr_conformance_matrix.glb"))
    for b in scene.bundles:   # (every fixture splat sits at (1, 2, 3): spread them out to see each one)
        k = scene.bundles.index(b)
        b.transform.matrix[:3, 3] = [(k % 5) * 0.6 - 1.2, (k // 5) * 0.6 - 0.6, 0.0]
        b.settings.global_scale = 0.3
    sh = plugin.add_scene(scene, f16=f16)
    handles, ref_entities = _oracle_entities(plugin, scene, f16)
    try:
        view = B.perspective_view((1, 2, 8), (1, 2, 3), 160, 96)
        got = plugin.render_entities(sh.entities(), view, fmt=fmt)
        want = plugin.render_entities(ref_entities, view, fmt=fmt)
        assert got.tobytes() == want.tobytes()
        assert np.any(got[..., 3] > 0)
    finally:
        sh.destroy()
        for h in handles:
            h.destroy()


def _two_camera_scene(n=3000):
    b = GltfBuilder()
    rng = np.random.default_rng(4)
    ids = []
    for m, combo in enumerate((CASE["rot_i8n"], CASE["sh2"])):
        arrays = primitive_arrays(combo, n, 20 + m)
        arrays[A_POS] = (rng.uniform(-2, 2, (n, 3)).astype(np.float32), False)
        arrays[A_SCALE] = (rng.uniform(-5, -2, (n, 3)).astype(np.float32), False)
        names = list(arrays)
        ids.append(b.mesh(dict(zip(names, b.accessors_of([arrays[k] for k in names], interleave=m == 1))),
                          {"kernel": "ellipse", "colorSpace": ["srgb_rec709_display", "lin_rec709_display"][m]}))
    child = b.node(root=False, name="inst", mesh=ids[0], translation=[0.5, 0.0, 0.0])
    b.node(name="a", mesh=ids[0], children=[child], scale=[0.5, 0.5, 0.5])
    b.node(name="b", mesh=ids[1], translation=[0.0, 0.3, -1.0])
    poses = [((0.5, 0.5, 6.0), (0.0, 0.0, 0.0)), ((-3.0, 1.0, 4.0), (0.0, 0.2, -0.5))]
    for j, (eye, target) in enumerate(poses):
        b.camera(f"cam{j}", np.linalg.inv(look_at_rh(eye, target, (0, 1, 0)).astype(np.float64)))
    return B.load_scene(b.glb()), poses


def test_views_match_per_view_frames(plugin):
    scene, poses = _two_camera_scene()
    assert len(scene.primitives) == 2 and len(scene.bundles) == 3
    sh = plugin.add_scene(scene)
    try:
        views = scene.views(128, 80)
        for v, (eye, target) in zip(views, poses):
            np.testing.assert_allclose(v.view_from_world, look_at_rh(eye, target, (0, 1, 0)), atol=1e-6)
        frames = plugin.render_views(sh.entities(), views)
        for f, v in zip(frames, views):
            assert f.tobytes() == plugin.render_entities(sh.entities(), v).tobytes()
            assert np.any(f[..., 3] > 0)
        handles, ref = _oracle_entities(plugin, scene, False)
        try:
            assert frames[0].tobytes() == plugin.render_entities(ref, views[0]).tobytes()
        finally:
            for h in handles:
                h.destroy()
    finally:
        sh.destroy()


def test_zero_quaternions_warn(plugin):
    scene = scene_of(primitive_arrays(COMBOS[0], 50, 1))
    with pytest.warns(UserWarning, match="zero-length quaternions"):
        sh = plugin.add_scene(scene)
    assert sh.zero_quats == [len(range(0, 50, 7))]
    sh.destroy()


def test_save_scene_round_trip(plugin, tmp_path):
    scene, _ = _two_camera_scene()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        sh = plugin.add_scene(scene)
    try:
        path = tmp_path / "saved.glb"
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            plugin.save_scene(path, sh.entities(), scene.cameras, names=[b.name for b in scene.bundles],
                              metadata=[b.metadata for b in scene.bundles])
            again = B.load_scene(path)
        assert len(again.bundles) == 3 and [c.name for c in again.cameras] == ["cam0", "cam1"]
        sh2 = plugin.add_scene(again)
        try:
            for v in scene.views(128, 80):
                a = plugin.render_entities(sh.entities(), v)
                b = plugin.render_entities(sh2.entities(), v)
                # the round trip moves scales by a few ulp (ln then exp) and rotations by one (normalised twice):
                # test_gpu_parity's bound for a cloud whose values moved by a rounding, and no drift on average
                assert float(np.abs(a - b).max()) <= ROUNDED_TOL and float(np.abs(a - b).mean()) <= 1e-5
        finally:
            sh2.destroy()
    finally:
        sh.destroy()
