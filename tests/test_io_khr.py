"""KHR_gaussian_splatting scenes on the host: the loader against the reference's conformance fixtures and its refusals,
buffers (data URIs, external files, interleaved and offset accessors), node hierarchies and instancing, the writer's
round trip, and the CPU restatement of the reference's attribute readers (khr_oracle)."""
import json
import os
import warnings

import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
from bevy_gaussian_splatting_b200.camera import look_at_rh
from khr_oracle import khr_oracle as K
from khr_cases import (A_COLOR, A_OP, A_POS, A_ROT, A_SCALE, COMBOS, EXT, GOLDEN, GltfBuilder, primitive_arrays,
                             scene_of, sh_name)

# khr_loader_conformance.rs:156-288: (scale_raw, opacity, sh_degree, colour space) per case
DEFAULT_SCALE, DEFAULT_OP = (0.0, 0.5, -0.5), 0.25
LIN, SRGB = B.GaussianColorSpace.LinRec709Display, B.GaussianColorSpace.SrgbRec709Display
EXPECTED = {name: (DEFAULT_SCALE, DEFAULT_OP, 0, LIN) for name in
            ("rotation_f32", "rotation_i8_norm", "rotation_i16_norm", "sh_degree0")}
EXPECTED.update({
    "scale_f32": ((0.2, -0.1, 0.7), DEFAULT_OP, 0, SRGB), "scale_i8": ((1.0, -2.0, 3.0), DEFAULT_OP, 0, LIN),
    "scale_i8_norm": ((1.0, 0.0, -1.0), DEFAULT_OP, 0, LIN), "scale_i16": ((2.0, -3.0, 4.0), DEFAULT_OP, 0, LIN),
    "scale_i16_norm": ((1.0, 0.0, -1.0), DEFAULT_OP, 0, LIN), "opacity_f32": (DEFAULT_SCALE, 0.75, 0, LIN),
    "opacity_u8_norm": (DEFAULT_SCALE, 64 / 255, 0, LIN), "opacity_u16_norm": (DEFAULT_SCALE, 16384 / 65535, 0, LIN),
    "sh_degree1": (DEFAULT_SCALE, DEFAULT_OP, 1, LIN), "sh_degree2": (DEFAULT_SCALE, DEFAULT_OP, 2, LIN),
    "sh_degree3": (DEFAULT_SCALE, DEFAULT_OP, 3, LIN)})


def load(path):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return B.load_scene(path)


@pytest.mark.parametrize("fixture", ["khr_conformance_matrix.gltf", "khr_conformance_matrix.glb"])
def test_conformance_matrix(fixture):
    scene = load(os.path.join(GOLDEN, fixture))
    assert len(scene.bundles) == 15 and len(scene.primitives) == 15
    assert [c.name for c in scene.cameras] == ["fixture_camera"]
    np.testing.assert_allclose(scene.cameras[0].matrix[:3, 3], [4, 5, 6], atol=1e-6)
    assert {b.name.split("_mesh")[0] for b in scene.bundles} == set(EXPECTED)
    for b in scene.bundles:
        scale_raw, opacity, degree, space = EXPECTED[b.name.split("_mesh")[0]]
        assert b.settings.color_space == space
        cloud, zero = K.decode(scene.primitives[b.primitive])
        assert zero == 0 and len(cloud) == 1 and cloud.sh_degree == degree
        np.testing.assert_allclose(cloud.position_visibility[0], [1, 2, 3, 1], atol=1e-6)
        np.testing.assert_allclose(cloud.rotation[0], [1, 0, 0, 0], atol=1e-5)
        np.testing.assert_allclose(cloud.scale_opacity[0, :3], np.exp(scale_raw), rtol=1e-5)
        np.testing.assert_allclose(cloud.scale_opacity[0, 3], opacity, atol=1e-5)
        for k in range((degree + 1) ** 2):
            np.testing.assert_allclose(cloud.spherical_harmonic[0, 3 * k:3 * k + 3], [k + 0.1, k + 0.2, k + 0.3], atol=1e-6)


def test_extensible_fallback_and_color0():
    with pytest.warns(UserWarning, match="customShape"):
        scene = B.load_scene(os.path.join(GOLDEN, "khr_extensible_fallback.gltf"))
    assert len(scene.bundles) == 1 and scene.cameras == []
    b = scene.bundles[0]
    assert b.settings.color_space == SRGB
    assert (b.metadata.kernel, b.metadata.color_space) == ("customShape", "custom_space_display")
    assert (b.metadata.projection, b.metadata.sorting_method) == ("perspective", "cameraDistance")
    assert b.metadata.extension_object["extensions"]["EXT_gaussian_splatting_kernel_customShape"] == {"gain": 1.25}
    cloud, _ = K.decode(scene.primitives[0])
    color = scene.primitives[0].color_0.array()[0, :3]
    np.testing.assert_array_equal(cloud.spherical_harmonic[0, :3], color / np.float32(0.282095))
    np.testing.assert_allclose(cloud.spherical_harmonic[0, :3], [1, 2, 3], atol=1e-4)
    assert cloud.scale_opacity[0, 3] == np.float32(0.5)
    root, _ = B.khr.encode_scene([B.SceneExportCloud(cloud, "extensible_unknown", b.settings, b.transform, b.metadata)])
    ext = root["meshes"][0]["primitives"][0]["extensions"][EXT]
    assert (ext["kernel"], ext["colorSpace"], ext["projection"], ext["sortingMethod"]) == \
        ("customShape", "custom_space_display", "perspective", "cameraDistance")
    assert ext["extensions"]["EXT_gaussian_splatting_kernel_customShape"] == {"gain": 1.25}


# ---- refusals

def _base(n=4):
    return primitive_arrays(COMBOS[0], n, 1)


def _refused(builder_fn, match):
    b = GltfBuilder()
    root = builder_fn(b)
    with pytest.raises(ValueError, match=match):
        B.load_scene(b.gltf(root))


def _one(b, arrays, ext=None, mode=0):
    names = list(arrays)
    b.node(name="n", mesh=b.mesh(dict(zip(names, b.accessors_of([arrays[k] for k in names]))), ext, mode))


def test_refuses_missing_extensions_used():
    _refused(lambda b: (_one(b, _base()), b.root(extensions_used=False))[1], "extensionsUsed")


def test_refuses_mode():
    _refused(lambda b: (_one(b, _base(), mode=4), b.root())[1], "mode")
    _refused(lambda b: (_one(b, _base(), mode=None), b.root())[1], "mode")


@pytest.mark.parametrize("missing", [A_POS, A_ROT, A_SCALE, A_OP])
def test_refuses_missing_attribute(missing):
    arrays = _base()
    del arrays[missing]
    _refused(lambda b: (_one(b, arrays), b.root())[1], "missing required attribute")


def test_refuses_count_mismatch():
    arrays = _base()
    arrays[A_OP] = (arrays[A_OP][0][:3], False)
    _refused(lambda b: (_one(b, arrays), b.root())[1], "entries; expected 4")


@pytest.mark.parametrize("coeffs,match", [
    ([(0, 0), (1, 0), (1, 1)], "partially defined"),          # degree 1 partial
    ([(0, 0)] + [(2, k) for k in range(5)], "degree 1 is required"),        # degree 1 skipped
    ([(1, k) for k in range(3)], "SH_DEGREE_0_COEF_0"),
    ([(0, 0)] + [(d, k) for d in (1, 2, 3, 4) for k in range(2 * d + 1)], "degree 4"),
])
def test_refuses_sh_maps(coeffs, match):
    arrays = _base()
    rng = np.random.default_rng(0)
    for d, k in coeffs:
        arrays[f"{EXT}:SH_DEGREE_{d}_COEF_{k}"] = (rng.uniform(-1, 1, (4, 3)).astype(np.float32), False)
    _refused(lambda b: (_one(b, arrays), b.root())[1], match)


def test_refuses_ranges_and_sparse():
    def accessor_past_view(b):
        _one(b, _base())
        b.accessors[0]["byteOffset"] = 4
        return b.root()

    def view_past_buffer(b):
        _one(b, _base())
        b.views[-1]["byteLength"] += 64
        return b.root()

    def sparse(b):
        _one(b, _base())
        b.accessors[2]["sparse"] = {"count": 1}
        return b.root()

    _refused(accessor_past_view, "lies outside bufferView")
    _refused(view_past_buffer, "lies outside buffer")
    _refused(sparse, "sparse")


def test_refuses_scene_without_splat_primitive():
    def unplaced(b):
        names = list(_base())
        b.mesh(dict(zip(names, b.accessors_of([_base()[k] for k in names]))))
        b.node(name="empty")
        return b.root()

    def no_primitives(b):
        b.node(name="empty")
        r = b.root()
        r["meshes"] = [{"primitives": [{"attributes": {}, "mode": 0}]}]
        return r

    _refused(unplaced, "no loadable gaussian primitives")
    _refused(no_primitives, "no KHR_gaussian_splatting primitives")


# ---- buffers and accessors

def test_percent_encoded_uri_and_external_bin(tmp_path):
    arrays = _base(3)
    b = GltfBuilder()
    _one(b, arrays)
    root = b.root()
    ref, _ = K.decode(B.load_scene(b.glb(root)).primitives[0])
    data = bytes(b.bin)
    # alphanumerics as themselves, every other byte as %XX in either case
    enc = "".join(chr(x) if chr(x).isalnum() and x < 0x80 else (f"%{x:02X}" if i % 2 else f"%{x:02x}") for i, x in enumerate(data))
    root["buffers"][0]["uri"] = "data:application/octet-stream," + enc
    got, _ = K.decode(B.load_scene(json.dumps(root).encode()).primitives[0])
    np.testing.assert_array_equal(got.scale_opacity, ref.scale_opacity)
    (tmp_path / "sub dir").mkdir()
    (tmp_path / "sub dir" / "splats data.bin").write_bytes(data)
    root["buffers"][0]["uri"] = "sub%20dir/splats%20data.bin"
    (tmp_path / "scene.gltf").write_text(json.dumps(root))
    got, _ = K.decode(B.load_scene(tmp_path / "scene.gltf").primitives[0])
    np.testing.assert_array_equal(got.rotation, ref.rotation)
    with pytest.raises(ValueError, match="external"):
        B.load_scene(json.dumps(root).encode())


@pytest.mark.parametrize("combo", COMBOS, ids=[c[0] for c in COMBOS])
def test_interleaved_and_offset_accessors_parse(combo):
    arrays = primitive_arrays(combo, 37, 3)
    packed = scene_of(arrays).primitives[0]
    for kw in (dict(interleave=True), dict(offset=12), dict(interleave=True, offset=8, container="gltf")):
        prim = scene_of(arrays, **kw).primitives[0]
        for name in ("position", "rotation", "scale", "opacity", "color_0"):
            a, b = getattr(packed, name), getattr(prim, name)
            if a is not None:
                np.testing.assert_array_equal(b.array(), a.array())
        ca, za = K.decode(packed)
        cb, zb = K.decode(prim)
        assert za == zb
        for pa, pb in zip((ca.position_visibility, ca.spherical_harmonic, ca.rotation, ca.scale_opacity),
                          (cb.position_visibility, cb.spherical_harmonic, cb.rotation, cb.scale_opacity)):
            np.testing.assert_array_equal(pa.view(np.uint32), pb.view(np.uint32))


def test_oracle_readers_follow_the_reference():
    f = np.float32
    q, zero = K.normalize_quaternions(np.array([[0, 0, 0, 0], [1e-4, 0, 0, 0], [3, 4, 0, 0], [2, 0, 0, 0]], f))
    assert zero == 2
    np.testing.assert_array_equal(q[:2], [[1, 0, 0, 0], [1, 0, 0, 0]])
    np.testing.assert_array_equal(q[2], np.array([3, 4, 0, 0], f) * (f(1) / np.sqrt(f(25))))
    b = GltfBuilder()
    arrays = _base(2)
    arrays[A_ROT] = (np.array([[-128, 127, 0, 0], [-127, 0, 0, 0]], np.int8), True)
    arrays[A_SCALE] = (np.array([[-32768, 32767, 0], [1, 2, 3]], np.int16), True)
    _one(b, arrays)
    prim = B.load_scene(b.gltf()).primitives[0]
    np.testing.assert_array_equal(K.read(prim.rotation)[0, :2], [-1.0, 1.0])   # max(v / 127, -1)
    np.testing.assert_array_equal(K.read(prim.scale)[0, :2], [-1.0, 1.0])
    assert K.read(prim.scale)[1, 0] == f(1) / f(32767)


# ---- nodes, instancing, cameras

def test_hierarchy_and_instancing():
    b = GltfBuilder()
    names = list(_base())
    mesh = b.mesh(dict(zip(names, b.accessors_of([_base()[k] for k in names]))))
    child_m = np.array([[0, -1, 0, 1], [1, 0, 0, 2], [0, 0, 1, 3], [0, 0, 0, 1]], np.float32)
    child = b.node(root=False, name="child", mesh=mesh, matrix=[float(v) for v in child_m.T.reshape(-1)])
    b.node(name="parent", translation=[10.0, 0.0, 0.0], scale=[2.0, 2.0, 2.0], children=[child])
    b.node(name="sibling", mesh=mesh)
    scene = B.load_scene(b.glb())
    assert len(scene.primitives) == 1
    assert [x.name for x in scene.bundles] == ["child_mesh0_primitive0", "sibling_mesh0_primitive0"]
    assert scene.bundles[0].primitive == scene.bundles[1].primitive == 0
    parent = np.diag([2, 2, 2, 1]).astype(np.float32)
    parent[0, 3] = 10
    np.testing.assert_array_equal(scene.bundles[0].transform.matrix, parent @ child_m)
    np.testing.assert_array_equal(scene.bundles[1].transform.matrix, np.eye(4))


def test_trs_rotation_matches_the_quaternion():
    b = GltfBuilder()
    _one(b, _base())
    s = np.sqrt(0.5)
    b.nodes[0].update(rotation=[0.0, 0.0, float(s), float(s)], translation=[1.0, 2.0, 3.0])   # 90 degrees about +z
    m = B.load_scene(b.gltf()).bundles[0].transform.matrix
    np.testing.assert_allclose(m, [[0, -1, 0, 1], [1, 0, 0, 2], [0, 0, 1, 3], [0, 0, 0, 1]], atol=1e-6)


def test_camera_views():
    b = GltfBuilder()
    _one(b, _base())
    eye, target = np.array([1.0, 0.5, 2.0]), np.array([0.0, 0.2, -1.0])
    v = look_at_rh(eye, target, (0, 1, 0))
    b.camera("cam", np.linalg.inv(v.astype(np.float64)))
    b.camera("ortho", np.eye(4), kind="orthographic")
    scene = B.load_scene(b.gltf())
    assert [c.name for c in scene.cameras] == ["cam", "ortho"]
    view = scene.cameras[0].view(64, 32)
    np.testing.assert_allclose(view.view_from_world, v, atol=1e-6)
    np.testing.assert_allclose(view.clip_from_view, B.camera.perspective_infinite_reverse_rh(0.8, 2.0, 0.05))
    with pytest.raises(ValueError, match="ortho"):
        scene.views(64, 32)


# ---- writer

def test_write_load_round_trip(tmp_path):
    cloud = B.random_gaussians_3d_seeded(500, 7, sh_degree=2)
    # scales in [0.25, 2]: ln then exp in f32 returns them within 2 ulp (an error that grows with |ln s| elsewhere)
    cloud.scale_opacity[:, :3] = np.float32(0.25) + cloud.scale_opacity[:, :3] * np.float32(1.75)
    cloud.rotation[17] = 0
    space = B.GaussianColorSpace.LinRec709Display
    meta = B.KhrSpec(kernel="customShape", sorting_method="byHash", extension_object={"extensions": {"EXT_x": {"a": 1}}})
    tr = B.CloudTransform(np.diag([1, 2, 3, 1]).astype(np.float32))
    cam = B.SceneCamera("eye", np.eye(4, dtype=np.float32), yfov=0.7, znear=0.02)
    keep = np.ones(500, bool)
    keep[17] = False
    for suffix in (".glb", ".gltf"):
        path = tmp_path / f"scene{suffix}"
        with pytest.warns(UserWarning, match="dropped 1 gaussians"):
            B.write_scene(path, [B.SceneExportCloud(cloud, "c0", B.CloudSettings(color_space=space), tr, meta)], [cam])
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            scene = B.load_scene(path)
        b = scene.bundles[0]
        assert b.name == "c0_mesh0_primitive0" and b.settings.color_space == space
        assert (b.metadata.kernel, b.metadata.sorting_method) == ("customShape", "byHash")
        assert b.metadata.extension_object["extensions"] == {"EXT_x": {"a": 1}}
        np.testing.assert_array_equal(b.transform.matrix, tr.matrix)
        assert scene.cameras[0].name == "eye" and scene.cameras[0].yfov == np.float32(0.7)
        got, zero = K.decode(scene.primitives[0])
        assert zero == 0 and len(got) == 499 and got.sh_degree == 2
        np.testing.assert_array_equal(got.position_visibility[:, :3], cloud.position_visibility[keep, :3])
        np.testing.assert_array_equal(got.spherical_harmonic, cloud.spherical_harmonic[keep])
        np.testing.assert_array_equal(got.scale_opacity[:, 3], cloud.scale_opacity[keep, 3])
        once, _ = K.normalize_quaternions(cloud.rotation[keep])
        np.testing.assert_array_equal(got.rotation, K.normalize_quaternions(once)[0])
        ulp = np.abs(got.scale_opacity[:, :3].view(np.int32) - cloud.scale_opacity[keep, :3].view(np.int32))
        assert ulp.max() <= 2
