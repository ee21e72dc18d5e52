"""Generated KHR_gaussian_splatting scenes for the loader's CPU tests and the GPU decode's parity tests: a small glTF
builder (tightly packed or interleaved bufferViews, accessor offsets, node hierarchies, cameras, .gltf or .glb) and
random attribute values for every (slot, component type, normalised) combination the reference accepts."""
from __future__ import annotations

import base64
import json
import os
import struct

import numpy as np

import bevy_gaussian_splatting_b200 as B

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "khr_gaussian_splatting")
EXT = "KHR_gaussian_splatting"
A_POS, A_ROT, A_SCALE, A_OP, A_COLOR = "POSITION", f"{EXT}:ROTATION", f"{EXT}:SCALE", f"{EXT}:OPACITY", "COLOR_0"
CTYPE = {np.dtype(np.int8): 5120, np.dtype(np.uint8): 5121, np.dtype(np.int16): 5122, np.dtype(np.uint16): 5123,
         np.dtype(np.float32): 5126}
KIND = {1: "SCALAR", 3: "VEC3", 4: "VEC4"}


def sh_name(k: int) -> str:
    d = int(np.sqrt(k))
    return f"{EXT}:SH_DEGREE_{d}_COEF_{k - d * d}"


class GltfBuilder:
    """Accessors of (n, c) numpy arrays in one buffer; meshes of one splat primitive each; nodes; cameras."""

    def __init__(self):
        self.bin = bytearray()
        self.views, self.accessors, self.meshes, self.nodes, self.cameras, self.roots = [], [], [], [], [], []

    def _pad(self):
        self.bin.extend(b"\0" * (-len(self.bin) % 4))

    def accessors_of(self, arrays, interleave: bool = False, offset: int = 0) -> list:
        """[(values, normalized)] -> accessor indices.  Packed: one bufferView each, the accessor `offset` bytes into it.
        Interleaved: one bufferView with every field 4-byte aligned, byteStride their sum, the accessors `offset` bytes in."""
        if not interleave:
            out = []
            for v, norm in arrays:
                self._pad()
                v = np.ascontiguousarray(v)
                self.views.append({"buffer": 0, "byteOffset": len(self.bin), "byteLength": offset + v.nbytes})
                self.bin.extend(b"\xAB" * offset + v.tobytes())
                out.append(self._accessor(v, norm, len(self.views) - 1, offset))
            return out
        fields, stride = [], 0
        for v, _ in arrays:
            fields.append(stride)
            stride += (v.dtype.itemsize * v.shape[1] + 3) & ~3
        n = len(arrays[0][0])
        rows = np.full((n, stride), 0xCD, np.uint8)
        for (v, _), f0 in zip(arrays, fields):
            w = v.dtype.itemsize * v.shape[1]
            rows[:, f0:f0 + w] = np.ascontiguousarray(v).view(np.uint8).reshape(n, w)
        self._pad()
        self.views.append({"buffer": 0, "byteOffset": len(self.bin), "byteLength": offset + rows.nbytes, "byteStride": stride})
        self.bin.extend(b"\xAB" * offset + rows.tobytes())
        return [self._accessor(v, norm, len(self.views) - 1, offset + f0) for (v, norm), f0 in zip(arrays, fields)]

    def _accessor(self, v, norm, view, offset):
        acc = {"bufferView": view, "byteOffset": offset, "componentType": CTYPE[v.dtype], "count": len(v), "type": KIND[v.shape[1]]}
        if norm:
            acc["normalized"] = True
        self.accessors.append(acc)
        return len(self.accessors) - 1

    def mesh(self, attributes: dict, ext=None, mode=0) -> int:
        prim = {"attributes": attributes, "extensions": {EXT: ext or {"kernel": "ellipse", "colorSpace": "lin_rec709_display"}}}
        if mode is not None:
            prim["mode"] = mode
        self.meshes.append({"primitives": [prim]})
        return len(self.meshes) - 1

    def node(self, root=True, **fields) -> int:
        self.nodes.append(fields)
        if root:
            self.roots.append(len(self.nodes) - 1)
        return len(self.nodes) - 1

    def camera(self, name, matrix, yfov=0.8, znear=0.05, kind="perspective") -> int:
        self.cameras.append({"type": kind, kind: {"yfov": yfov, "znear": znear, "zfar": 100.0} if kind == "perspective"
                             else {"xmag": 1.0, "ymag": 1.0, "znear": znear, "zfar": 100.0}})
        return self.node(name=name, camera=len(self.cameras) - 1, matrix=[float(x) for x in np.asarray(matrix, np.float32).T.reshape(-1)])

    def root(self, extensions_used=True) -> dict:
        self._pad()
        r = {"asset": {"version": "2.0"}, "scene": 0, "scenes": [{"nodes": self.roots}], "nodes": self.nodes,
             "meshes": self.meshes, "buffers": [{"byteLength": len(self.bin)}], "bufferViews": self.views,
             "accessors": self.accessors}
        if extensions_used:
            r["extensionsUsed"] = [EXT]
        if self.cameras:
            r["cameras"] = self.cameras
        return r

    def gltf(self, root=None) -> bytes:
        r = root or self.root()
        r["buffers"][0]["uri"] = "data:application/octet-stream;base64," + base64.b64encode(bytes(self.bin)).decode()
        return json.dumps(r).encode()

    def glb(self, root=None) -> bytes:
        js = json.dumps(root or self.root()).encode()
        js += b" " * (-len(js) % 4)
        binary = bytes(self.bin)
        return (struct.pack("<4sII", b"glTF", 2, 28 + len(js) + len(binary)) + struct.pack("<II", len(js), 0x4E4F534A) + js
                + struct.pack("<II", len(binary), 0x004E4942) + binary)


# ---- attribute values

def values(slot: str, dtype, normalized: bool, n: int, rng, comps=None) -> np.ndarray:
    """Random accepted values of one slot; rotations include zero-length rows (and, quantised, rows that round to zero)."""
    dt = np.dtype(dtype)
    c = comps or {"pos": 3, "rot": 4, "scale": 3, "op": 1, "color": 3, "sh": 3}[slot]
    if dt == np.float32:
        lo, hi = {"pos": (-20, 20), "rot": (-1, 1), "scale": (-4, 1), "op": (0, 1), "color": (0, 1), "sh": (-1, 1)}[slot]
        v = rng.uniform(lo, hi, (n, c)).astype(np.float32)
    elif slot == "scale" and not normalized:
        v = rng.integers(-12, 4, (n, c)).astype(dt)
    else:
        info = np.iinfo(dt)
        v = rng.integers(info.min, int(info.max) + 1, (n, c)).astype(dt)
    if slot == "rot":
        v[::7] = 0
    return v


DEFAULT = {"pos": (np.float32, False), "rot": (np.float32, False), "scale": (np.float32, False), "op": (np.float32, False)}
# every accepted combination, one slot varied from the f32 default at a time: (id, slot, dtype, normalised, components)
COMBOS = ([("rot_f32", "rot", np.float32, False, 4), ("rot_i8n", "rot", np.int8, True, 4), ("rot_i16n", "rot", np.int16, True, 4)]
          + [(f"scale_{t.__name__}{'n' if nm else ''}", "scale", t, nm, 3) for t in (np.int8, np.int16) for nm in (False, True)]
          + [("op_u8n", "op", np.uint8, True, 1), ("op_u16n", "op", np.uint16, True, 1)]
          + [(f"color{c}_f32", "color", np.float32, False, c) for c in (3, 4)]
          + [(f"color{c}_{t.__name__}{'n' if nm else ''}", "color", t, nm, c) for c in (3, 4) for t in (np.uint8, np.uint16)
             for nm in (False, True)]
          + [(f"sh{d}", "sh", np.float32, False, d) for d in range(4)])


def primitive_arrays(combo, n: int, seed: int) -> dict:
    """{attribute semantic: (values, normalised)} of one COMBOS case."""
    _, slot, dtype, norm, extra = combo
    rng = np.random.default_rng(seed)
    spec = dict(DEFAULT)
    if slot in spec:
        spec[slot] = (dtype, norm)
    out = {A_POS: (values("pos", *spec["pos"], n, rng), False), A_ROT: (values("rot", *spec["rot"], n, rng), spec["rot"][1]),
           A_SCALE: (values("scale", *spec["scale"], n, rng), spec["scale"][1]), A_OP: (values("op", *spec["op"], n, rng), spec["op"][1])}
    if slot == "color":
        out[A_COLOR] = (values("color", dtype, norm, n, rng, comps=extra), norm)
    elif slot == "sh":
        for k in range((extra + 1) ** 2):
            out[sh_name(k)] = (values("sh", np.float32, False, n, rng), False)
    return out


def scene_of(arrays: dict, interleave=False, offset=0, container="glb", ext=None) -> B.GaussianScene:
    """One node placing one primitive of `arrays`, loaded back through B.load_scene."""
    b = GltfBuilder()
    names = list(arrays)
    idx = b.accessors_of([arrays[k] for k in names], interleave, offset)
    b.node(name="n0", mesh=b.mesh(dict(zip(names, idx)), ext))
    return B.load_scene(b.glb() if container == "glb" else b.gltf())
