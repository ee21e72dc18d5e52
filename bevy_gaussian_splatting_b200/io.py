"""Input formats for the path (SURVEY.md §8 row f1): INRIA-style 3DGS `.ply` -> PlanarGaussian3d.

Restates src/io/ply.rs:23-132 of the reference, including its quirks:
  * opacity = sigmoid(raw)                                   ply.rs:40-42
  * scale_i = exp(clamp(raw_i, mean(raw) -+ 4))              ply.rs:103-116 (MAX_SIZE_VARIANCE = 4)
  * rotation normalised (w, x, y, z = rot_0..3)              ply.rs:118-124
  * f_rest_i -> channel = i / 16 (not i / 15), coefficient = (i % 15) + 1, interleaved index
    coefficient * 3 + channel, ignored when >= 48            ply.rs:49-69 (later properties overwrite earlier)
    At SH degree d (the reference's sh_d build; K_d = (d + 1)^2, S_d = 4, 12, 28, 48): channel = i / K_d, coefficient
    = 1 if K_d == 1 else (i % (K_d - 1)) + 1, kept when coefficient * 3 + channel < S_d -- so sh0 stores f_rest_0 in
    padding lane 3.
  * the cloud is padded with default gaussians by 32 - (n % 32) entries -- a full 32 when n is already
    a multiple of 32                                          ply.rs:127-129
`.gcloud` (flexbuffers serde, src/io/gcloud/flexbuffers.rs:9-22) lives in `gcloud.py`; `load_cloud` below is the
extension switch of the reference's asset loader (src/io/loader.rs:38-66).
"""
from __future__ import annotations

import io
import os

import numpy as np

from .gaussian import PlanarGaussian3d, PlanarGaussian4d, SH_4D_COEFF_COUNT, SH_WIDTHS, sh_bands

MAX_SIZE_VARIANCE = 4.0
SH_CHANNELS = 3
REQUIRED = ["x", "y", "z", "f_dc_0", "f_dc_1", "f_dc_2", "scale_0", "scale_1", "opacity", "rot_0", "rot_1", "rot_2", "rot_3"]
_PLY_TYPES = {"float": "f4", "float32": "f4", "double": "f8", "float64": "f8", "uchar": "u1", "uint8": "u1", "char": "i1",
              "int8": "i1", "short": "i2", "int16": "i2", "ushort": "u2", "uint16": "u2", "int": "i4", "int32": "i4",
              "uint": "u4", "uint32": "u4"}


def _read_header(f):
    if f.readline().strip() != b"ply":
        raise ValueError("not a PLY file")
    fmt, elements, cur = None, [], None
    while True:
        line = f.readline()
        if not line:
            raise ValueError("unterminated PLY header")
        tok = line.decode("ascii", "replace").split()
        if not tok:
            continue
        if tok[0] == "format":
            fmt = tok[1]
        elif tok[0] == "element":
            cur = {"name": tok[1], "count": int(tok[2]), "props": []}
            elements.append(cur)
        elif tok[0] == "property":
            if tok[1] == "list":     # (count type, item type): fine in other elements (faces), skipped with them
                if cur["name"] == "vertex":
                    raise ValueError("list properties are not supported in the vertex element")
                cur["props"].append((tok[4], ("list", _PLY_TYPES[tok[2]], _PLY_TYPES[tok[3]])))
            else:
                cur["props"].append((tok[2], _PLY_TYPES[tok[1]]))
        elif tok[0] == "end_header":
            break
    return fmt, elements


def parse_ply_3d(source, sh_degree: int = 3) -> PlanarGaussian3d:
    """`source`: path, bytes or binary file object.  A malformed file raises ValueError (ply.rs returns io::Error).
    `sh_degree`: the SH degree of the cloud made (the reference's sh0 .. sh3 builds), f_rest_ placed by its rule."""
    if sh_degree not in range(4):
        raise ValueError(f"sh_degree must be 0..3, not {sh_degree}")
    if isinstance(source, (str, os.PathLike)):
        with open(source, "rb") as fh:
            return parse_ply_3d(fh.read(), sh_degree)
    try:
        with np.errstate(over="ignore", invalid="ignore"):
            return _parse_ply_3d(source, sh_degree)
    except (TypeError, IndexError, KeyError, UnicodeDecodeError, OverflowError, MemoryError) as e:
        raise ValueError(f"malformed ply: {type(e).__name__}: {e}") from e


def _parse_ply_3d(source, sh_degree: int) -> PlanarGaussian3d:
    width, bands = SH_WIDTHS[sh_degree], sh_bands(sh_degree)
    f = io.BytesIO(source) if isinstance(source, (bytes, bytearray)) else source
    fmt, elements = _read_header(f)
    vertex = None
    for el in elements:
        if el["name"] == "vertex":
            missing = [k for k in REQUIRED if k not in [p for p, _ in el["props"]]]
            if missing:
                raise ValueError("missing required properties")     # ply.rs:92-97
            if fmt == "ascii":
                rows = np.loadtxt(f, dtype=np.float64, max_rows=el["count"], ndmin=2)
                vertex = {p: rows[:, i].astype(np.float32) for i, (p, _) in enumerate(el["props"])}
            else:
                end = "<" if fmt == "binary_little_endian" else ">"
                dt = np.dtype([(p, end + t) for p, t in el["props"]])
                raw = np.frombuffer(f.read(dt.itemsize * el["count"]), dtype=dt, count=el["count"])
                vertex = {p: raw[p] for p, t in el["props"] if t == "f4"}   # only Property::Float is consumed
        else:
            if fmt == "ascii":
                for _ in range(el["count"]):
                    f.readline()
            else:
                end = "<" if fmt == "binary_little_endian" else ">"
                if any(isinstance(t, tuple) for _, t in el["props"]):
                    for _ in range(el["count"]):            # rows with list properties have no fixed stride
                        for _, t in el["props"]:
                            if isinstance(t, tuple):
                                cnt = int(np.frombuffer(f.read(np.dtype(t[1]).itemsize), end + t[1], 1)[0])
                                f.read(cnt * np.dtype(t[2]).itemsize)
                            else:
                                f.read(np.dtype(t).itemsize)
                else:
                    f.read(np.dtype([(p, end + t) for p, t in el["props"]]).itemsize * el["count"])
    if vertex is None:
        return PlanarGaussian3d(np.zeros((0, 4), np.float32), np.zeros((0, width), np.float32), np.zeros((0, 4), np.float32),
                                np.zeros((0, 4), np.float32))
    n = len(vertex["x"])
    pos = np.zeros((n, 4), np.float32); pos[:, 3] = 1.0                # PositionVisibility::default: visibility 1
    sh = np.zeros((n, width), np.float32)
    rot = np.zeros((n, 4), np.float32)
    so = np.zeros((n, 4), np.float32)
    for key, v in vertex.items():                                      # header order, like set_property calls
        v = v.astype(np.float32)
        if key in ("x", "y", "z"):
            pos[:, "xyz".index(key)] = v
        elif key == "visibility":
            pos[:, 3] = v
        elif key in ("f_dc_0", "f_dc_1", "f_dc_2"):
            sh[:, int(key[-1])] = v
        elif key in ("scale_0", "scale_1", "scale_2"):
            so[:, int(key[-1])] = v
        elif key == "opacity":
            so[:, 3] = np.float32(1.0) / (np.float32(1.0) + np.exp(-v))
        elif key in ("rot_0", "rot_1", "rot_2", "rot_3"):
            rot[:, int(key[-1])] = v
        elif key.startswith("f_rest_"):
            i = int(key[7:])
            channel = i // bands
            coefficient = 1 if bands == 1 else (i % (bands - 1)) + 1
            idx = coefficient * SH_CHANNELS + channel
            if idx < width:
                sh[:, idx] = v
    mean = (so[:, 0] + so[:, 1] + so[:, 2]) / np.float32(3.0)
    for i in range(3):
        so[:, i] = np.exp(np.minimum(np.maximum(so[:, i], mean - np.float32(MAX_SIZE_VARIANCE)), mean + np.float32(MAX_SIZE_VARIANCE)))
    norm = np.sqrt((rot.astype(np.float32) ** 2).sum(axis=1, dtype=np.float32))
    with np.errstate(invalid="ignore", divide="ignore"):
        rot = (rot / norm[:, None]).astype(np.float32)
    pad = 32 - (n % 32)
    def padded(a, fill_last=None):
        z = np.zeros((pad, a.shape[1]), np.float32)
        if fill_last is not None:
            z[:, -1] = fill_last
        return np.concatenate([a, z])
    return PlanarGaussian3d(padded(pos, 1.0), padded(sh), padded(rot), padded(so))


def write_ply_3d(path, cloud: PlanarGaussian3d, n: int | None = None) -> None:
    """Test helper: the inverse transformation (logit opacity, log scale, INRIA property order).  A degree-d cloud
    writes 3 (K_d - 1) f_rest_ properties, channel-major (none at degree 0); its padding lanes are not written."""
    n = len(cloud) if n is None else n
    rest = sh_bands(cloud.sh_degree) - 1   # coefficients per channel beyond the DC term
    props = ["x", "y", "z", "nx", "ny", "nz", "f_dc_0", "f_dc_1", "f_dc_2"] + [f"f_rest_{i}" for i in range(3 * rest)] + \
            ["opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"]
    arr = np.zeros(n, np.dtype([(p, "<f4") for p in props]))
    arr["x"], arr["y"], arr["z"] = cloud.position_visibility[:n, 0], cloud.position_visibility[:n, 1], cloud.position_visibility[:n, 2]
    for c in range(3):
        arr[f"f_dc_{c}"] = cloud.spherical_harmonic[:n, c]
    for i in range(3 * rest):   # INRIA planar order: channel-major, K_d - 1 coefficients each
        arr[f"f_rest_{i}"] = cloud.spherical_harmonic[:n, ((i % rest) + 1) * 3 + i // rest]
    o = np.clip(cloud.scale_opacity[:n, 3].astype(np.float64), 1e-6, 1 - 1e-6)
    arr["opacity"] = np.log(o / (1 - o)).astype(np.float32)
    for c in range(3):
        arr[f"scale_{c}"] = np.log(np.maximum(cloud.scale_opacity[:n, c], 1e-12))
    for c in range(4):
        arr[f"rot_{c}"] = cloud.rotation[:n, c]
    with open(path, "wb") as f:
        f.write(("ply\nformat binary_little_endian 1.0\nelement vertex %d\n" % n).encode())
        for p in props:
            f.write(f"property float {p}\n".encode())
        f.write(b"end_header\n")
        f.write(arr.tobytes())


# ply.rs:134-182: the float properties of a Gaussian4d vertex -> (plane, column)
PLY4D_PROPERTIES = {"x": (0, 0), "y": (0, 1), "z": (0, 2), "visibility": (0, 3), "t": (4, 0), "st": (4, 1),
                    "sx": (3, 0), "sy": (3, 1), "sz": (3, 2), "opacity": (3, 3),
                    "rot_x": (2, 0), "rot_y": (2, 1), "rot_z": (2, 2), "rot_w": (2, 3),
                    "rot_r_x": (2, 4), "rot_r_y": (2, 5), "rot_r_z": (2, 6), "rot_r_w": (2, 7)}
PLY4D_REQUIRED = ["x", "y", "z", "t", "st", "sx", "sy", "sz", "opacity", "rot_x", "rot_y", "rot_z", "rot_w",
                  "rot_r_x", "rot_r_y", "rot_r_z", "rot_r_w"]


def parse_ply_4d(source) -> PlanarGaussian4d:
    """ply.rs:134-247, `parse_ply_4d`: float properties only (others are ignored, as the reference's match ignores
    them); feat_{r,g,b}_{i} -> coefficient 3 i + channel (ignored past 144); the required properties above or
    ValueError; both quaternions divided by their norms, lanes in the file's rot_x, rot_y, rot_z, rot_w order (lane 0,
    read by the shader as w, is rot_x); padded with default gaussians (visibility 1, all else 0) by 32 - (n % 32)."""
    if isinstance(source, (str, os.PathLike)):
        with open(source, "rb") as fh:
            return parse_ply_4d(fh.read())
    try:
        return _parse_ply_4d(source)
    except (TypeError, IndexError, KeyError, UnicodeDecodeError, OverflowError, MemoryError) as e:
        raise ValueError(f"malformed ply4d: {type(e).__name__}: {e}") from e


def _parse_ply_4d(source) -> PlanarGaussian4d:
    f = io.BytesIO(source) if isinstance(source, (bytes, bytearray)) else source
    fmt, elements = _read_header(f)
    if fmt != "binary_little_endian":
        raise ValueError(f"only binary_little_endian PLY is supported, got {fmt}")
    planes = [np.zeros((0, w), np.float32) for w in (4, SH_4D_COEFF_COUNT, 8, 4, 4)]
    for el in elements:
        if any(isinstance(t, tuple) for _, t in el["props"]):
            raise ValueError("list properties are not supported")
        dt = np.dtype([(name, "<" + t) for name, t in el["props"]])
        data = np.frombuffer(f.read(dt.itemsize * el["count"]), dt, count=el["count"])
        if el["name"] != "vertex":
            continue
        names = [name for name, _ in el["props"]]
        if any(r not in names for r in PLY4D_REQUIRED):
            raise ValueError("missing required properties")
        n = el["count"]
        planes = [np.zeros((n, w), np.float32) for w in (4, SH_4D_COEFF_COUNT, 8, 4, 4)]
        planes[0][:, 3] = 1.0
        for name, t in el["props"]:
            if t != "f4":
                continue
            if name in PLY4D_PROPERTIES:
                k, c = PLY4D_PROPERTIES[name]
                planes[k][:, c] = data[name]
            elif name.startswith("feat_"):
                channel = "rgb".index(name[5])
                idx = int(name[7:]) * 3 + channel
                if idx < SH_4D_COEFF_COUNT:
                    planes[1][:, idx] = data[name]
    rot = planes[2]
    with np.errstate(invalid="ignore", divide="ignore"):
        for lo in (0, 4):
            q = rot[:, lo:lo + 4]
            norm = np.sqrt(np.sum(q * q, axis=1, dtype=np.float32), dtype=np.float32)
            rot[:, lo:lo + 4] = (q / norm[:, None]).astype(np.float32)
    pad = 32 - (len(rot) % 32)
    out = []
    for k, a in enumerate(planes):
        z = np.zeros((pad, a.shape[1]), np.float32)
        if k == 0:
            z[:, 3] = 1.0
        out.append(np.concatenate([a, z]))
    return PlanarGaussian4d(*out)


def write_ply_4d(path, cloud: PlanarGaussian4d, n: int | None = None) -> None:
    """The first n gaussians of `cloud` as a binary .ply4d `parse_ply_4d` reads back (every property float)."""
    n = len(cloud) if n is None else n
    props = list(PLY4D_PROPERTIES) + [f"feat_{'rgb'[i % 3]}_{i // 3}" for i in range(SH_4D_COEFF_COUNT)]
    arr = np.zeros(n, np.dtype([(p, "<f4") for p in props]))
    planes = cloud.planes()
    for name, (k, c) in PLY4D_PROPERTIES.items():
        arr[name] = planes[k][:n, c]
    for i in range(SH_4D_COEFF_COUNT):
        arr[f"feat_{'rgb'[i % 3]}_{i // 3}"] = planes[1][:n, i]
    with open(path, "wb") as f:
        f.write(("ply\nformat binary_little_endian 1.0\nelement vertex %d\n" % n).encode())
        for p in props:
            f.write(f"property float {p}\n".encode())
        f.write(b"end_header\n")
        f.write(arr.tobytes())


def load_cloud(path) -> PlanarGaussian3d | PlanarGaussian4d:
    """`Gaussian3dLoader::load` (src/io/loader.rs:24-70): `.ply` -> parse_ply_3d, `.gcloud` -> CloudCodec::decode;
    `Gaussian4dLoader::load` (loader.rs:69-115): `.ply4d` -> parse_ply_4d (`.gc4d` is not read here); anything else is
    an error."""
    ext = os.path.splitext(str(path))[1].lower()
    if ext == ".ply4d":
        return parse_ply_4d(path)
    if ext == ".ply":
        return parse_ply_3d(path)
    if ext == ".gcloud":
        from .gcloud import read_gcloud

        return read_gcloud(path)
    raise ValueError("only .ply and .gcloud supported")
