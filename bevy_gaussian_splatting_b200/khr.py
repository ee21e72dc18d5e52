"""KHR_gaussian_splatting glTF / GLB scenes: the reference's scene loader and writer (src/io/scene.rs).

`load_scene` restates `load_gltf_scene` / `collect_gaussian_primitives` / `collect_node_bundles` (scene.rs:288-765) on the
host: it parses the container, the buffers, the extension objects, the node hierarchy and the cameras, and describes
each placed primitive's attributes as typed, strided accessors into the buffers it holds.  It never decodes a gaussian:
`GaussianSplattingPlugin.add_scene` hands the descriptors to `bgs_cloud_upload_khr`, which copies each accessor's span
once and decodes it on the GPU.  `write_scene` restates `encode_khr_gaussian_scene_gltf_bytes` / `_glb_bytes`
(scene.rs:766-1130) for host clouds.  Sparse accessors are refused (the reference's glTF reader would apply them).
"""
from __future__ import annotations

import base64
import dataclasses
import json
import math
import os
import re
import struct
import urllib.parse
import warnings

import numpy as np

from . import abi
from .camera import View, perspective_infinite_reverse_rh
from .gaussian import PlanarGaussian3d, sh_bands
from .plugin import CloudTransform
from .settings import CloudSettings, GaussianColorSpace, GaussianMode

EXTENSION = "KHR_gaussian_splatting"
ATTR_POSITION, ATTR_COLOR_0 = "POSITION", "COLOR_0"
ATTR_ROTATION, ATTR_SCALE, ATTR_OPACITY = (f"{EXTENSION}:ROTATION", f"{EXTENSION}:SCALE", f"{EXTENSION}:OPACITY")
SH_SEMANTIC = re.compile(re.escape(f"{EXTENSION}:SH_DEGREE_") + r"(\d+)_COEF_(\d+)$")
COMPONENT_DTYPES = {5120: np.int8, 5121: np.uint8, 5122: np.int16, 5123: np.uint16, 5125: np.uint32, 5126: np.float32}
TYPE_COMPONENTS = {"SCALAR": 1, "VEC2": 2, "VEC3": 3, "VEC4": 4, "MAT2": 4, "MAT3": 9, "MAT4": 16}
COLOR_SPACES = {"srgb_rec709_display": GaussianColorSpace.SrgbRec709Display,
                "lin_rec709_display": GaussianColorSpace.LinRec709Display}
# (field, extension key, known values, fallback): scene.rs:451-554
SPEC_FIELDS = (("kernel", "kernel", ("ellipse",), "ellipse"),
               ("color_space", "colorSpace", tuple(COLOR_SPACES), "srgb_rec709_display"),
               ("projection", "projection", ("perspective",), "perspective"),
               ("sorting_method", "sortingMethod", ("cameraDistance",), "cameraDistance"))
GLB_MAGIC, GLB_JSON, GLB_BIN = b"glTF", 0x4E4F534A, 0x004E4942


@dataclasses.dataclass
class KhrAccessor:
    """One attribute's accessor: `count` elements of `components` values of glTF type `component_type`, element 0 at
    `offset` bytes into `buffer`, `stride` bytes apart (the bufferView's byteStride, or the element size)."""

    buffer: memoryview
    offset: int
    stride: int
    component_type: int
    normalized: bool
    components: int
    count: int

    def array(self) -> np.ndarray:
        """The (count, components) strided view of the buffer (no copy)."""
        dt = np.dtype(COMPONENT_DTYPES[self.component_type])
        return np.ndarray((self.count, self.components), dt, buffer=self.buffer, offset=self.offset,
                          strides=(self.stride, dt.itemsize))

    def to_abi(self) -> abi.bgs_khr_accessor:
        base = np.frombuffer(self.buffer, np.uint8).ctypes.data
        return abi.bgs_khr_accessor(data=base + self.offset, byte_stride=self.stride, component_type=self.component_type,
                                    normalized=int(self.normalized), components=self.components)


@dataclasses.dataclass
class KhrSpec:
    """The primitive's extension values as written (GaussianPrimitiveSpec) and the extension object itself, kept for
    export; unknown values render as ellipse / srgb_rec709_display / perspective / cameraDistance."""

    kernel: str = "ellipse"
    color_space: str = "srgb_rec709_display"
    projection: str = "perspective"
    sorting_method: str = "cameraDistance"
    extension_object: dict | None = None


@dataclasses.dataclass
class KhrPrimitive:
    """One splat primitive (mesh, primitive) some node of the scene places: its accessors, SH degree and extension."""

    mesh: int
    primitive: int
    n: int
    position: KhrAccessor
    rotation: KhrAccessor
    scale: KhrAccessor
    opacity: KhrAccessor
    color_0: KhrAccessor | None
    sh: list           # KhrAccessor per coefficient d*d + c, (sh_degree + 1)^2 of them, or [] (no SH)
    sh_degree: int
    spec: KhrSpec
    color_space: GaussianColorSpace

    def to_abi(self) -> abi.bgs_khr_primitive:
        p = abi.bgs_khr_primitive(n=self.n, position=self.position.to_abi(), rotation=self.rotation.to_abi(),
                                  scale=self.scale.to_abi(), opacity=self.opacity.to_abi(), sh_degree=self.sh_degree)
        if self.color_0 is not None:
            p.color_0 = self.color_0.to_abi()
        for k, a in enumerate(self.sh):
            p.sh[k] = a.to_abi()
        return p


@dataclasses.dataclass
class SceneBundle:
    """A placed primitive (CloudBundle): name "{node}_mesh{m}_primitive{p}", the index of its primitive in
    `GaussianScene.primitives`, its CloudSettings, its node's world matrix and the primitive's extension values."""

    name: str
    primitive: int
    settings: CloudSettings
    transform: CloudTransform
    metadata: KhrSpec


@dataclasses.dataclass
class SceneCamera:
    """A camera node: its name, world matrix (row-major numpy, f32) and glTF camera values.  Also the writer's camera."""

    name: str
    matrix: np.ndarray = dataclasses.field(default_factory=lambda: np.eye(4, dtype=np.float32))
    type: str = "perspective"
    yfov: float = math.pi / 4
    znear: float = 0.01
    zfar: float | None = 1000.0

    def view(self, width: int, height: int) -> View:
        """The camera's View: view_from_world the inverse of its world matrix (glTF and Bevy both look down -Z, +Y up),
        perspective_infinite_reverse_rh(yfov, width / height, znear); zfar and aspectRatio are not applied."""
        if self.type != "perspective":
            raise ValueError(f"camera '{self.name}' is {self.type}: only perspective cameras give a view")
        m = np.asarray(self.matrix, np.float64)
        return View(np.linalg.inv(m).astype(np.float32), perspective_infinite_reverse_rh(self.yfov, width / height, self.znear),
                    m[:3, 3].astype(np.float32), int(width), int(height))


@dataclasses.dataclass
class GaussianScene:
    primitives: list
    bundles: list
    cameras: list
    buffers: list = dataclasses.field(default_factory=list, repr=False)   # what the accessors point into

    def views(self, width: int, height: int) -> list:
        """One View per camera, in the scene's order; an orthographic camera raises ValueError naming it."""
        return [c.view(width, height) for c in self.cameras]


# ---- reading

def _split_glb(data: memoryview) -> tuple[dict, memoryview | None]:
    if len(data) < 12:
        raise ValueError("GLB: shorter than its 12-byte header")
    _, version, length = struct.unpack_from("<4sII", data, 0)
    if version != 2 or length > len(data):
        raise ValueError(f"GLB: version {version}, length {length} of {len(data)} bytes")
    pos, js, bin_ = 12, None, None
    while pos + 8 <= length:
        clen, ctype = struct.unpack_from("<II", data, pos)
        if pos + 8 + clen > length:
            raise ValueError("GLB: a chunk runs past the file")
        chunk = data[pos + 8:pos + 8 + clen]
        if ctype == GLB_JSON and js is None:
            js = json.loads(bytes(chunk))
        elif ctype == GLB_BIN and bin_ is None:
            bin_ = chunk
        pos += 8 + ((clen + 3) & ~3)
    if js is None:
        raise ValueError("GLB: no JSON chunk")
    return js, bin_


def _decode_data_uri(uri: str) -> bytes:
    """scene.rs:615-686: base64 when a ';base64' part is present, else percent-decoded."""
    meta, sep, payload = uri[5:].partition(",")
    if not sep:
        raise ValueError("malformed data URI; expected a ',' separator")
    if any(part.lower() == "base64" for part in meta.split(";")):
        return base64.b64decode(payload, validate=True)
    out, i, b = bytearray(), 0, payload.encode()
    while i < len(b):
        if b[i] == 0x25:   # '%'
            hexd = b[i + 1:i + 3]
            if len(hexd) < 2 or i + 2 >= len(b) or not all(c in b"0123456789abcdefABCDEF" for c in hexd):
                raise ValueError("malformed percent-encoded data URI payload")
            out.append(int(hexd, 16))
            i += 3
        else:
            out.append(b[i])
            i += 1
    return bytes(out)


def _load_buffers(root: dict, bin_chunk, base_dir) -> list:
    out = []
    for j, buf in enumerate(root.get("buffers", [])):
        uri = buf.get("uri")
        if uri is None:
            if bin_chunk is None:
                raise ValueError(f"buffer {j} references the BIN chunk but there is none")
            data, bin_chunk = bin_chunk, None
        elif uri.startswith("data:"):
            data = memoryview(_decode_data_uri(uri))
        else:
            if base_dir is None:
                raise ValueError(f"buffer {j} is the external file '{uri}', but the scene was given as bytes")
            with open(os.path.join(base_dir, urllib.parse.unquote(uri)), "rb") as f:
                data = memoryview(f.read())
        if len(data) < int(buf.get("byteLength", 0)):
            raise ValueError(f"buffer {j} length mismatch: expected at least {buf.get('byteLength')} bytes, got {len(data)}")
        out.append(data)
    return out


def _accessor(root: dict, buffers: list, index: int, semantic: str) -> KhrAccessor:
    accessors = root.get("accessors", [])
    if not 0 <= index < len(accessors):
        raise ValueError(f"attribute semantic '{semantic}' references missing accessor index {index}")
    acc = accessors[index]
    if "sparse" in acc:
        raise ValueError(f"attribute semantic '{semantic}': sparse accessors are not supported")
    if "bufferView" not in acc:
        raise ValueError(f"attribute semantic '{semantic}': accessor {index} has no bufferView")
    ctype, kind, count = int(acc["componentType"]), acc["type"], int(acc["count"])
    if ctype not in COMPONENT_DTYPES or kind not in TYPE_COMPONENTS:
        raise ValueError(f"attribute semantic '{semantic}': componentType {ctype} / type {kind} is not a glTF accessor type")
    views = root.get("bufferViews", [])
    vi = int(acc["bufferView"])
    if not 0 <= vi < len(views):
        raise ValueError(f"attribute semantic '{semantic}' references missing bufferView {vi}")
    view = views[vi]
    bi = int(view["buffer"])
    if not 0 <= bi < len(buffers):
        raise ValueError(f"bufferView {vi} references missing buffer {bi}")
    comps = TYPE_COMPONENTS[kind]
    elem = np.dtype(COMPONENT_DTYPES[ctype]).itemsize * comps
    stride = int(view.get("byteStride", elem))
    v_off, v_len, a_off = int(view.get("byteOffset", 0)), int(view["byteLength"]), int(acc.get("byteOffset", 0))
    if v_off < 0 or v_len < 0 or v_off + v_len > len(buffers[bi]):
        raise ValueError(f"bufferView {vi} ([{v_off}, {v_off + v_len})) lies outside buffer {bi} ({len(buffers[bi])} bytes)")
    span = (count - 1) * stride + elem if count > 0 else 0
    if a_off < 0 or stride < elem or a_off + span > v_len:
        raise ValueError(f"attribute semantic '{semantic}': accessor {index} ({count} x {stride} B from {a_off}) lies outside "
                         f"bufferView {vi} ({v_len} bytes)")
    return KhrAccessor(buffers[bi], v_off + a_off, stride, ctype, bool(acc.get("normalized", False)), comps, count)


def _sh_map(attributes: dict) -> tuple[int, list]:
    """collect_sh_coefficient_map (scene.rs:1457-1550): (degree, accessor indices by coefficient d*d + c), or (0, [])."""
    degrees: dict[int, dict[int, int]] = {}
    for semantic, index in attributes.items():
        m = SH_SEMANTIC.match(semantic)
        if m:
            degrees.setdefault(int(m.group(1)), {})[int(m.group(2))] = int(index)
    if not degrees:
        return 0, []
    if 0 not in degrees.get(0, {}):
        raise ValueError(f"missing required spherical harmonics attribute '{EXTENSION}:SH_DEGREE_0_COEF_0'")
    top = max(degrees)
    if top > 3:
        raise ValueError(f"unsupported spherical harmonics degree {top}; KHR_gaussian_splatting supports degrees up to 3")
    out = []
    for d in range(top + 1):
        coeffs = degrees.get(d)
        if coeffs is None:
            raise ValueError(f"spherical harmonics degree {d} is required because higher degrees are present, but its "
                             "coefficients are missing")
        if sorted(coeffs) != list(range(2 * d + 1)):
            raise ValueError(f"spherical harmonics degree {d} is partially defined; it must define exactly coefficients "
                             f"0..{2 * d}")
        out += [coeffs[c] for c in range(2 * d + 1)]
    return top, out


def _spec(ext, mesh: int, prim: int) -> KhrSpec:
    if not isinstance(ext, dict):
        raise ValueError(f"mesh {mesh} primitive {prim} has an invalid KHR_gaussian_splatting extension payload")
    values = {}
    for field, key, known, fallback in SPEC_FIELDS:
        v = ext.get(key, fallback if key in ("projection", "sortingMethod") else None)
        if not isinstance(v, str):
            raise ValueError(f"mesh {mesh} primitive {prim} has an invalid KHR_gaussian_splatting extension payload: "
                             f"{key} is missing or not a string")
        if not v.strip():
            raise ValueError(f"mesh {mesh} primitive {prim} has an empty KHR_gaussian_splatting {key} value")
        if v not in known:
            warnings.warn(f"mesh {mesh} primitive {prim} uses extension {key} '{v}'; falling back to '{fallback}'")
        values[field] = v
    return KhrSpec(**values, extension_object=ext)


def _node_matrix(node: dict) -> np.ndarray:
    """The node's local matrix, row-major f32: `matrix` (column-major in the file), or T * R * S as glam's
    from_scale_rotation_translation builds it."""
    f = np.float32
    if "matrix" in node:
        return np.asarray(node["matrix"], f).reshape(4, 4).T.copy()
    x, y, z, w = (f(v) for v in node.get("rotation", (0.0, 0.0, 0.0, 1.0)))
    s = np.asarray(node.get("scale", (1.0, 1.0, 1.0)), f)
    t = np.asarray(node.get("translation", (0.0, 0.0, 0.0)), f)
    x2, y2, z2 = x + x, y + y, z + z
    xx, xy, xz, yy, yz, zz = x * x2, x * y2, x * z2, y * y2, y * z2, z * z2
    wx, wy, wz = w * x2, w * y2, w * z2
    one = f(1.0)
    cols = [np.array([one - (yy + zz), xy + wz, xz - wy], f) * s[0], np.array([xy - wz, one - (xx + zz), yz + wx], f) * s[1],
            np.array([xz + wy, yz - wx, one - (xx + yy)], f) * s[2]]
    m = np.eye(4, dtype=f)
    for c in range(3):
        m[:3, c] = cols[c]
    m[:3, 3] = t
    return m


def load_scene(path_or_bytes) -> GaussianScene:
    """A `.gltf` / `.glb` KHR_gaussian_splatting scene (a path, or the file's bytes; GLB is found by its magic).  Every
    refusal is a ValueError; unknown extension values fall back with a warning."""
    base_dir = None
    if isinstance(path_or_bytes, (bytes, bytearray, memoryview)):
        data = memoryview(path_or_bytes)
    else:
        with open(path_or_bytes, "rb") as f:
            data = memoryview(f.read())
        base_dir = os.path.dirname(os.path.abspath(path_or_bytes))
    if bytes(data[:4]) == GLB_MAGIC:
        root, bin_chunk = _split_glb(data)
    else:
        try:
            root, bin_chunk = json.loads(bytes(data)), None
        except (UnicodeDecodeError, json.JSONDecodeError) as e:
            raise ValueError(f"failed to parse glTF JSON: {e}") from None

    # collect_gaussian_primitives (scene.rs:387-449)
    sources = {}
    for mi, mesh in enumerate(root.get("meshes", [])):
        for pi, prim in enumerate(mesh.get("primitives", [])):
            ext = prim.get("extensions", {}).get(EXTENSION)
            if ext is None:
                continue
            mode = prim.get("mode", 4)
            if mode != 0:
                raise ValueError(f"mesh {mi} primitive {pi} has KHR_gaussian_splatting but mode={mode}; mode must be POINTS (0)")
            sources[(mi, pi)] = (prim.get("attributes", {}), _spec(ext, mi, pi))
    if not sources:
        raise ValueError("no KHR_gaussian_splatting primitives found")
    if EXTENSION not in root.get("extensionsUsed", []):
        raise ValueError("KHR_gaussian_splatting primitives are present but the extension is missing from extensionsUsed")
    buffers = _load_buffers(root, bin_chunk, base_dir)
    scenes = root.get("scenes", [])
    if not scenes:
        raise ValueError("glTF does not contain any scenes")
    scene = scenes[int(root.get("scene", 0))]
    nodes, meshes, cams = root.get("nodes", []), root.get("meshes", []), root.get("cameras", [])

    primitives, index_of, bundles, cameras = [], {}, [], []

    def primitive(mi: int, pi: int) -> int:
        if (mi, pi) not in index_of:
            attributes, spec = sources[(mi, pi)]

            def required(semantic):
                if semantic not in attributes:
                    raise ValueError(f"missing required attribute semantic '{semantic}'")
                return _accessor(root, buffers, int(attributes[semantic]), semantic)

            pos, rot, scale, op = (required(s) for s in (ATTR_POSITION, ATTR_ROTATION, ATTR_SCALE, ATTR_OPACITY))
            degree, sh_idx = _sh_map(attributes)
            sh = [_accessor(root, buffers, a, f"{EXTENSION}:SH") for a in sh_idx]
            color = None
            if not sh and ATTR_COLOR_0 in attributes:
                color = _accessor(root, buffers, int(attributes[ATTR_COLOR_0]), ATTR_COLOR_0)
            n = pos.count
            for name, a in [(ATTR_ROTATION, rot), (ATTR_SCALE, scale), (ATTR_OPACITY, op), (ATTR_COLOR_0, color)] + \
                    [(f"{EXTENSION}:SH_{k}", a) for k, a in enumerate(sh)]:
                if a is not None and a.count != n:
                    raise ValueError(f"attribute semantic '{name}' has {a.count} entries; expected {n}")
            index_of[(mi, pi)] = len(primitives)
            primitives.append(KhrPrimitive(mi, pi, n, pos, rot, scale, op, color, sh, degree, spec,
                                           COLOR_SPACES.get(spec.color_space, GaussianColorSpace.SrgbRec709Display)))
        return index_of[(mi, pi)]

    # collect_node_bundles (scene.rs:688-764): depth first, a node's camera and primitives before its children
    def visit(ni: int, parent: np.ndarray, path: tuple):
        if not 0 <= ni < len(nodes) or ni in path:
            raise ValueError(f"node {ni} is missing or its own ancestor")
        node = nodes[ni]
        world = (parent @ _node_matrix(node)).astype(np.float32)
        name = node.get("name") or "gaussian_node"
        if "camera" in node:
            cam = cams[int(node["camera"])]
            kind = cam.get("type", "perspective")
            p = cam.get(kind, {})
            cameras.append(SceneCamera(name, world, kind, float(p.get("yfov", math.pi / 4)), float(p.get("znear", 0.01)),
                                       None if p.get("zfar") is None else float(p["zfar"])))
        if "mesh" in node:
            mi = int(node["mesh"])
            for pi in range(len(meshes[mi].get("primitives", []))):
                if (mi, pi) not in sources:
                    continue
                j = primitive(mi, pi)
                prim = primitives[j]
                settings = CloudSettings(gaussian_mode=GaussianMode.Gaussian3d, color_space=prim.color_space)
                bundles.append(SceneBundle(f"{name}_mesh{mi}_primitive{pi}", j, settings, CloudTransform(world.copy()), prim.spec))
        for child in node.get("children", []):
            visit(int(child), world, path + (ni,))

    for ni in scene.get("nodes", []):
        visit(int(ni), np.eye(4, dtype=np.float32), ())
    if not bundles:
        raise ValueError("KHR_gaussian_splatting scene contained no loadable gaussian primitives")
    return GaussianScene(primitives, bundles, cameras, buffers)


# ---- writing

@dataclasses.dataclass
class SceneExportCloud:
    """One cloud `write_scene` writes (the reference's SceneExportCloud): a host cloud, its name, settings (color_space
    is written), transform (its matrix is the node's) and the extension values to keep (None: the defaults)."""

    cloud: PlanarGaussian3d
    name: str
    settings: CloudSettings = dataclasses.field(default_factory=CloudSettings)
    transform: CloudTransform | None = None
    metadata: KhrSpec | None = None


def _extension_object(meta: KhrSpec | None, color_space) -> dict:
    """gaussian_extension_object (scene.rs:1185-1259): the kept object with each value the spec's when it is an unknown
    (extension) value, else the one the settings render with."""
    meta = meta or KhrSpec()
    obj = dict(meta.extension_object or {})
    current = {"kernel": "ellipse", "color_space": "lin_rec709_display" if int(color_space) == GaussianColorSpace.LinRec709Display
               else "srgb_rec709_display", "projection": "perspective", "sorting_method": "cameraDistance"}
    for field, key, known, _ in SPEC_FIELDS:
        v = getattr(meta, field).strip()
        obj[key] = current[field] if not v or v in known else v
    return obj


def encode_scene(bundles, cameras=()) -> tuple[dict, bytes]:
    """(glTF JSON, binary buffer) of `bundles` (SceneExportCloud) and `cameras` (SceneCamera), every accessor f32."""
    f = np.float32
    binary, views, accessors, meshes, nodes, scene_nodes, cams_json = bytearray(), [], [], [], [], [], []

    def push(values: np.ndarray, kind: str, lo=None, hi=None) -> int:
        binary.extend(b"\0" * (-len(binary) % 4))
        views.append({"buffer": 0, "byteOffset": len(binary), "byteLength": values.nbytes})
        binary.extend(np.ascontiguousarray(values, "<f4").tobytes())
        acc = {"bufferView": len(views) - 1, "componentType": 5126, "count": len(values), "type": kind}
        if lo is not None:
            acc["min"], acc["max"] = [float(v) for v in lo], [float(v) for v in hi]
        accessors.append(acc)
        return len(accessors) - 1

    for b in bundles:
        c = b.cloud
        if len(c) == 0:
            continue
        q = c.rotation
        l2 = ((q[:, 0] * q[:, 0] + q[:, 1] * q[:, 1]) + q[:, 2] * q[:, 2]) + q[:, 3] * q[:, 3]
        keep = (l2 > np.finfo(f).eps) & np.isfinite(l2)
        if not keep.any():
            warnings.warn(f"skipping cloud '{b.name}' during KHR export because all gaussians had invalid rotations")
            continue
        if not keep.all():
            warnings.warn(f"dropped {int((~keep).sum())} gaussians with invalid rotations while exporting cloud '{b.name}'")
        inv = (f(1.0) / np.sqrt(l2[keep])).astype(f)
        pos = c.position_visibility[keep, :3]
        with np.errstate(divide="ignore"):
            scale = np.log(np.maximum(c.scale_opacity[keep, :3], f(1e-6))).astype(f)
        attrs = {ATTR_POSITION: push(pos, "VEC3", pos.min(0), pos.max(0)),
                 ATTR_ROTATION: push((q[keep] * inv[:, None]).astype(f), "VEC4"),
                 ATTR_SCALE: push(scale, "VEC3"),
                 ATTR_OPACITY: push(np.clip(c.scale_opacity[keep, 3], f(0.0), f(1.0)), "SCALAR")}
        sh = c.spherical_harmonic[keep]
        for k in range(sh_bands(c.sh_degree)):
            d = int(math.isqrt(k))
            attrs[f"{EXTENSION}:SH_DEGREE_{d}_COEF_{k - d * d}"] = push(sh[:, 3 * k:3 * k + 3], "VEC3")
        ext = _extension_object(b.metadata, b.settings.color_space)
        meshes.append({"name": b.name, "primitives": [{"attributes": attrs, "mode": 0, "extensions": {EXTENSION: ext}}]})
        m = np.eye(4, dtype=f) if b.transform is None else np.asarray(b.transform.matrix, f)
        scene_nodes.append(len(nodes))
        nodes.append({"name": b.name, "mesh": len(meshes) - 1, "matrix": [float(v) for v in m.T.reshape(-1)]})
    if not scene_nodes:
        raise ValueError("cannot export a KHR_gaussian_splatting scene with zero gaussians")
    for cam in cameras:
        persp = {"yfov": float(f(cam.yfov)), "znear": float(f(cam.znear))}
        if cam.zfar is not None:
            persp["zfar"] = float(f(cam.zfar))
        cams_json.append({"name": cam.name, "type": "perspective", "perspective": persp})
        scene_nodes.append(len(nodes))
        nodes.append({"name": cam.name, "camera": len(cams_json) - 1,
                      "matrix": [float(v) for v in np.asarray(cam.matrix, f).T.reshape(-1)]})
    binary.extend(b"\0" * (-len(binary) % 4))
    root = {"asset": {"version": "2.0"}, "extensionsUsed": [EXTENSION], "extensionsRequired": [EXTENSION], "scene": 0,
            "scenes": [{"nodes": scene_nodes}], "nodes": nodes, "meshes": meshes,
            "buffers": [{"byteLength": len(binary)}], "bufferViews": views, "accessors": accessors}
    if cams_json:
        root["cameras"] = cams_json
    return root, bytes(binary)


def write_scene(path, bundles, cameras=()) -> None:
    """Write `bundles` (SceneExportCloud) and `cameras` (SceneCamera) as a KHR_gaussian_splatting scene: `.glb` with a
    BIN chunk, `.gltf` with the buffer embedded as base64.  What the reference's exporter writes: f32 accessors,
    ln(max(scale, 1e-6)), opacity clamped to [0, 1], normalised rotations (gaussians whose rotation is zero-length or
    non-finite are dropped), SH up to each cloud's degree, one node per cloud with its matrix, and the camera nodes."""
    ext = os.path.splitext(str(path))[1].lower()
    if ext not in (".gltf", ".glb"):
        raise ValueError("write_scene: the path must end in .gltf or .glb")
    root, binary = encode_scene(bundles, cameras)
    if ext == ".gltf":
        root["buffers"][0]["uri"] = "data:application/octet-stream;base64," + base64.b64encode(binary).decode()
        out = json.dumps(root, indent=2).encode()
    else:
        js = json.dumps(root, separators=(",", ":")).encode()
        js += b" " * (-len(js) % 4)
        out = (struct.pack("<4sII", GLB_MAGIC, 2, 12 + 8 + len(js) + 8 + len(binary)) + struct.pack("<II", len(js), GLB_JSON) + js
               + struct.pack("<II", len(binary), GLB_BIN) + binary)
    with open(path, "wb") as fh:
        fh.write(out)
