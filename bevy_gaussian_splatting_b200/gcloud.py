"""`.gcloud` codec for the path's input row f1 (SURVEY.md §8f): `CloudCodec::encode / decode` of the reference
(src/io/codec.rs:4-18, src/io/gcloud/flexbuffers.rs:9-22) = the serde serialisation of `PlanarGaussian3d` into a
FlexBuffer, uncompressed (src/io/loader.rs: `Some("gcloud") => PlanarGaussian3d::decode(bytes)`).

The encoding itself lives in two crates that are NOT in the reference repository (`flexbuffers` 25.2 and the `Planar` derive
of `bevy_interleave`), so this module restates the published FlexBuffers wire format (google/flatbuffers
`flexbuffers.h`: values are read from the END of the buffer; offsets point backwards; vectors carry a length prefix and,
when untyped, one packed-type byte per element; maps are a vector of values plus a sorted key vector) and serde's data
model for the structs involved:

    PlanarGaussian3d { position_visibility: Vec<PositionVisibility>, spherical_harmonic: Vec<SphericalHarmonicCoefficients>,
                       rotation: Vec<Rotation>, scale_opacity: Vec<ScaleOpacity> }            planar_3d.rs:45-54
    PositionVisibility { position: [f32; 3], visibility: f32 }                                f32.rs:53-56
    SphericalHarmonicCoefficients { coefficients: [f32; 48] }  (serialised as a 48-tuple)     spherical_harmonics.rs:114-120
    Rotation { rotation: [f32; 4] }                                                           f32.rs:95-97
    ScaleOpacity { scale: [f32; 3], opacity: f32 }                                            f32.rs:172-175

struct -> map keyed by field name, Vec / array / tuple -> vector.  The READER is generic (any valid FlexBuffer: every
scalar width, typed / fixed-typed / untyped vectors, maps, indirect scalars), so it does not depend on which of the
equivalent encodings a writer picked.  The reference pins this format only through a round trip
(tests/io.rs:7-17, tests/gaussian.rs: `decode(encode(random_gaussians_3d(n))) == original`); that is the bar held here
too (tests/test_io_gcloud.py).  **Parity with bytes written by the Rust crate is unpinned**: no reference-written
`.gcloud` file exists in this image.
"""
from __future__ import annotations

import struct

import numpy as np

from .gaussian import SH_WIDTHS, PlanarGaussian3d

# FlexBuffers value types (flexbuffers.h, enum Type)
FBT_NULL, FBT_INT, FBT_UINT, FBT_FLOAT, FBT_KEY, FBT_STRING = 0, 1, 2, 3, 4, 5
FBT_INDIRECT_INT, FBT_INDIRECT_UINT, FBT_INDIRECT_FLOAT = 6, 7, 8
FBT_MAP, FBT_VECTOR, FBT_VECTOR_INT, FBT_VECTOR_UINT, FBT_VECTOR_FLOAT, FBT_VECTOR_KEY = 9, 10, 11, 12, 13, 14
FBT_VECTOR_STRING_DEPRECATED = 15
FBT_VECTOR_INT2, FBT_VECTOR_FLOAT4 = 16, 24      # 16..24: fixed-length typed vectors (INT2, UINT2, FLOAT2, INT3, ...)
FBT_BLOB, FBT_BOOL, FBT_VECTOR_BOOL = 25, 26, 36

_UFMT = {1: "<B", 2: "<H", 4: "<I", 8: "<Q"}
_IFMT = {1: "<b", 2: "<h", 4: "<i", 8: "<q"}
_FDT = {4: "<f4", 8: "<f8"}


class FlexBufferError(ValueError):
    pass


# ----------------------------------------------------------------------------------------------- reader
class Ref:
    """A value inside a FlexBuffer: (buffer, position of the value or of its offset, width of that slot, packed type)."""

    __slots__ = ("buf", "pos", "parent_width", "type", "byte_width")

    def __init__(self, buf, pos: int, parent_width: int, packed: int):
        if pos < 0 or pos + parent_width > len(buf):
            raise FlexBufferError("value outside the buffer")
        self.buf, self.pos, self.parent_width = buf, pos, parent_width
        self.type, self.byte_width = packed >> 2, 1 << (packed & 3)

    # -- low level
    def _u(self, pos: int, width: int) -> int:
        if pos < 0 or pos + width > len(self.buf):
            raise FlexBufferError("read outside the buffer")
        return struct.unpack_from(_UFMT[width], self.buf, pos)[0]

    def _target(self) -> int:
        t = self.pos - self._u(self.pos, self.parent_width)
        if t < 0 or t > len(self.buf):
            raise FlexBufferError("offset outside the buffer")
        return t

    # -- scalars
    def as_float(self) -> float:
        if self.type == FBT_FLOAT:
            pos, w = self.pos, self.parent_width
        elif self.type == FBT_INDIRECT_FLOAT:
            pos, w = self._target(), self.byte_width
        elif self.type in (FBT_INT, FBT_UINT, FBT_INDIRECT_INT, FBT_INDIRECT_UINT, FBT_BOOL):
            return float(self.as_int())
        elif self.type == FBT_NULL:
            return 0.0
        else:
            raise FlexBufferError(f"type {self.type} is not a number")
        if w not in _FDT:
            raise FlexBufferError(f"float of width {w}")
        return float(np.frombuffer(self.buf, _FDT[w], 1, pos)[0])

    def as_int(self) -> int:
        if self.type in (FBT_INT, FBT_UINT, FBT_BOOL):
            pos, w = self.pos, self.parent_width
        elif self.type in (FBT_INDIRECT_INT, FBT_INDIRECT_UINT):
            pos, w = self._target(), self.byte_width
        elif self.type in (FBT_FLOAT, FBT_INDIRECT_FLOAT):
            return int(self.as_float())
        elif self.type == FBT_NULL:
            return 0
        else:
            raise FlexBufferError(f"type {self.type} is not a number")
        fmt = _IFMT if self.type in (FBT_INT, FBT_INDIRECT_INT) else _UFMT
        return struct.unpack_from(fmt[w], self.buf, pos)[0]

    def as_key(self) -> bytes:
        if self.type not in (FBT_KEY, FBT_STRING):
            raise FlexBufferError("not a key / string")
        t = self._target()
        if self.type == FBT_STRING:
            return bytes(self.buf[t:t + self._u(t - self.byte_width, self.byte_width)])
        end = self.buf.find(b"\0", t) if isinstance(self.buf, (bytes, bytearray)) else bytes(self.buf[t:]).find(b"\0") + t
        if end < 0:
            raise FlexBufferError("unterminated key")
        return bytes(self.buf[t:end])

    # -- vectors
    def is_vector(self) -> bool:
        return self.type in (FBT_MAP, FBT_VECTOR, FBT_VECTOR_BOOL) or FBT_VECTOR_INT <= self.type <= FBT_VECTOR_FLOAT4

    def _vector_info(self):
        """(position of element 0, length, element type or None when untyped)."""
        t = self._target()
        ty = self.type
        if FBT_VECTOR_INT2 <= ty <= FBT_VECTOR_FLOAT4:
            return t, (ty - FBT_VECTOR_INT2) // 3 + 2, (ty - FBT_VECTOR_INT2) % 3 + FBT_INT
        n = self._u(t - self.byte_width, self.byte_width)
        if ty in (FBT_VECTOR, FBT_MAP):
            return t, n, None
        if ty == FBT_VECTOR_BOOL:
            return t, n, FBT_BOOL
        if FBT_VECTOR_INT <= ty <= FBT_VECTOR_STRING_DEPRECATED:
            return t, n, ty - FBT_VECTOR_INT + FBT_INT
        raise FlexBufferError(f"type {ty} is not a vector")

    def __len__(self) -> int:
        return self._vector_info()[1]

    def __getitem__(self, i: int) -> "Ref":
        t, n, ety = self._vector_info()
        if not 0 <= i < n:
            raise IndexError(i)
        w = self.byte_width
        if ety is None:
            packed = self._u(t + n * w + i, 1)
        else:
            packed = (ety << 2) | {1: 0, 2: 1, 4: 2, 8: 3}[w]      # typed: children are scalars / keys of this width
        return Ref(self.buf, t + i * w, w, packed)

    def as_float_array(self) -> np.ndarray:
        """Any vector of numbers -> float32 array (typed float vectors are read in one piece)."""
        t, n, ety = self._vector_info()
        w = self.byte_width
        if ety == FBT_FLOAT and w in _FDT:
            if t + n * w > len(self.buf):
                raise FlexBufferError("vector outside the buffer")
            return np.frombuffer(self.buf, _FDT[w], n, t).astype(np.float32)
        return np.array([self[i].as_float() for i in range(n)], np.float32)

    # -- maps
    def keys(self) -> list[bytes]:
        if self.type != FBT_MAP:
            raise FlexBufferError("not a map")
        t = self._target()
        w = self.byte_width
        kpos = t - 3 * w
        kvec = kpos - self._u(kpos, w)
        kw = self._u(t - 2 * w, w)
        n = self._u(kvec - kw, kw)
        return [Ref(self.buf, kvec + i * kw, kw, (FBT_KEY << 2)).as_key() for i in range(n)]

    def as_dict(self) -> dict:
        ks = self.keys()
        return {k: self[i] for i, k in enumerate(ks)}


def root(data) -> Ref:
    buf = data if isinstance(data, (bytes, bytearray)) else bytes(data)
    if len(buf) < 3:
        raise FlexBufferError("buffer too small")
    width = buf[-1]
    if width not in (1, 2, 4, 8) or len(buf) < 2 + width:
        raise FlexBufferError("bad root width")
    return Ref(buf, len(buf) - 2 - width, width, buf[-2])


# ----------------------------------------------------------------------------------------------- writer
class Builder:
    """Minimal FlexBuffers writer (children first, offsets backwards): 32-bit floats, float vectors, maps, vectors.
    Every offset / length slot is 4 bytes wide (buffers below 4 GiB), which any conforming reader accepts."""

    W = 4

    def __init__(self):
        self.out = bytearray()
        self._keys: dict[bytes, int] = {}
        self._keyvecs: dict[tuple, int] = {}

    def _align(self):
        self.out += b"\0" * (-len(self.out) % self.W)

    def key(self, k: bytes) -> int:
        pos = self._keys.get(k)
        if pos is None:
            pos = len(self.out)
            self.out += k + b"\0"
            self._keys[k] = pos
        return pos

    def float_vector(self, values: np.ndarray):
        """-> (position of element 0, packed type).  2..4 elements use the fixed-length typed vector (no length)."""
        v = np.ascontiguousarray(values, "<f4").reshape(-1)
        self._align()
        n = len(v)
        if 2 <= n <= 4:
            ty = FBT_VECTOR_INT2 + (n - 2) * 3 + (FBT_FLOAT - FBT_INT)
        else:
            ty = FBT_VECTOR_FLOAT
            self.out += struct.pack("<I", n)
        pos = len(self.out)
        self.out += v.tobytes()
        return pos, (ty << 2) | 2

    def _slots(self, items):
        """items: list of ('f', float) | ('o', position, packed) -> value slots + type bytes, written at the current end."""
        types = bytearray()
        for it in items:
            if it[0] == "f":
                self.out += struct.pack("<f", it[1])
                types.append((FBT_FLOAT << 2) | 2)
            else:
                off = len(self.out) - it[1]
                if off <= 0 or off >= 1 << 32:
                    raise FlexBufferError("offset does not fit 32 bits")
                self.out += struct.pack("<I", off)
                types.append(it[2])
        self.out += types

    def vector(self, items):
        self._align()
        self.out += struct.pack("<I", len(items))
        pos = len(self.out)
        self._slots(items)
        return pos, (FBT_VECTOR << 2) | 2

    def map(self, entries: dict):
        """entries: {key bytes: item}; keys sorted bytewise (strcmp order), key vectors shared between equal key sets."""
        ks = tuple(sorted(entries))
        kv = self._keyvecs.get(ks)
        if kv is None:
            kpos = [self.key(k) for k in ks]
            self._align()
            self.out += struct.pack("<I", len(ks))
            kv = len(self.out)
            for p in kpos:
                self.out += struct.pack("<I", len(self.out) - p)
            self._keyvecs[ks] = kv
        self._align()
        self.out += struct.pack("<I", len(self.out) - kv)      # offset to the key vector
        self.out += struct.pack("<I", self.W)                  # its byte width
        self.out += struct.pack("<I", len(ks))
        pos = len(self.out)
        self._slots([entries[k] for k in ks])
        return pos, (FBT_MAP << 2) | 2

    def finish(self, pos: int, packed: int) -> bytes:
        self._align()
        self.out += struct.pack("<I", len(self.out) - pos)
        self.out += bytes([packed, self.W])
        return bytes(self.out)


# ----------------------------------------------------------------------------------------------- the cloud codec
_PLANES = (
    # plane of PlanarGaussian3d, [(field, first column, width)] of its element struct
    (b"position_visibility", "position_visibility", ((b"position", 0, 3), (b"visibility", 3, 1))),
    (b"spherical_harmonic", "spherical_harmonic", ((b"coefficients", 0, 48),)),   # (S_d at degree d: _sh_fields)
    (b"rotation", "rotation", ((b"rotation", 0, 4),)),
    (b"scale_opacity", "scale_opacity", ((b"scale", 0, 3), (b"opacity", 3, 1))),
)


def _sh_fields(width: int):
    """The SH plane's fields for an S_d-tuple (the reference's sh_d build serialises [f32; S_d])."""
    return ((b"coefficients", 0, width),)


def _cloud_planes(cloud: PlanarGaussian3d):
    """_PLANES with the SH plane at the cloud's width."""
    return tuple((key, attr, _sh_fields(cloud.spherical_harmonic.shape[1]) if attr == "spherical_harmonic" else fields)
                 for key, attr, fields in _PLANES)


def _sh_width(pr: "Ref") -> int:
    """The S_d of an SH plane, from its first element's coefficient tuple (4, 12, 28 or 48; 48 for an empty plane or an
    element that leaves the field to its default).  Any other length raises FlexBufferError."""
    if len(pr) == 0:
        return 48
    e = pr[0]
    if e.type == FBT_MAP:
        v = e.as_dict().get(b"coefficients")
    elif e.is_vector():
        v = e[0] if len(e) else None
    else:
        raise FlexBufferError("plane element is not a struct")
    if v is None:
        return 48
    w = len(v.as_float_array())
    if w not in SH_WIDTHS:
        raise FlexBufferError(f"coefficients has {w} elements, expected 4, 12, 28 or 48 (SH degree 0..3)")
    return w


def _encode_plane(b: Builder, arr: np.ndarray, fields):
    """All N element structs of one plane at once (numpy), in the same layout Builder.map / float_vector produce one
    by one: per element [its float vectors][key-vector offset, key width, length][one slot per field][type bytes, pad].
    Returns the plane's ("o", position, packed) item."""
    n = len(arr)
    ks = tuple(sorted(fk for fk, _, _ in fields))
    by_key = {fk: (c0, w) for fk, c0, w in fields}
    # the shared key vector (written once, before the elements)
    kpos = [b.key(k) for k in ks]
    b._align()
    b.out += struct.pack("<I", len(ks))
    kv = len(b.out)
    for p in kpos:
        b.out += struct.pack("<I", len(b.out) - p)
    b._keyvecs.setdefault(ks, kv)
    b._align()
    base = len(b.out)
    # record layout
    rec, off, vec_at = [], 0, {}
    for fk in ks:
        c0, w = by_key[fk]
        if w > 1:
            if not 2 <= w <= 4:
                rec.append((f"l_{fk.decode()}", "<u4")); off += 4                  # length prefix of a VECTOR_FLOAT
            vec_at[fk] = off
            rec.append((f"v_{fk.decode()}", "<f4", (w,))); off += 4 * w
    hdr_at = off
    rec += [("koff", "<u4"), ("kw", "<u4"), ("len", "<u4")]; off += 12
    slot_at = {}
    for fk in ks:
        slot_at[fk] = off
        rec.append((f"s_{fk.decode()}", "<f4" if by_key[fk][1] == 1 else "<u4")); off += 4
    rec.append(("types", "u1", (len(ks),))); off += len(ks)
    pad = -off % 4
    if pad:
        rec.append(("pad", "u1", (pad,))); off += pad
    dt = np.dtype(rec)
    assert dt.itemsize == off
    r = np.zeros(n, dt)
    idx = np.arange(n, dtype=np.int64)
    rec_pos = base + idx * off
    koff = rec_pos + hdr_at - kv
    if n and int(koff.max()) >= 1 << 32:
        raise FlexBufferError("offset does not fit 32 bits")
    r["koff"], r["kw"], r["len"] = koff, Builder.W, len(ks)
    types = []
    for fk in ks:
        c0, w = by_key[fk]
        name = fk.decode()
        if w == 1:
            r[f"s_{name}"] = arr[:, c0]
            types.append((FBT_FLOAT << 2) | 2)
        else:
            r[f"v_{name}"] = arr[:, c0:c0 + w]
            if 2 <= w <= 4:
                ty = FBT_VECTOR_INT2 + (w - 2) * 3 + (FBT_FLOAT - FBT_INT)
            else:
                ty = FBT_VECTOR_FLOAT
                r[f"l_{name}"] = w
            r[f"s_{name}"] = slot_at[fk] - vec_at[fk]                  # constant backwards distance inside the record
            types.append((ty << 2) | 2)
    r["types"] = np.array(types, np.uint8)
    b.out += r.tobytes()
    # the plane: an untyped vector of N maps
    b._align()
    b.out += struct.pack("<I", n)
    pos = len(b.out)
    first_value = rec_pos + hdr_at + 12                                # a map is referenced by its first value slot
    slots = pos + 4 * idx - first_value
    if n and int(slots.max()) >= 1 << 32:
        raise FlexBufferError("offset does not fit 32 bits")
    b.out += slots.astype("<u4").tobytes()
    b.out += bytes([(FBT_MAP << 2) | 2]) * n
    return ("o", pos, (FBT_VECTOR << 2) | 2)


def encode_gcloud_elementwise(cloud: PlanarGaussian3d) -> bytes:
    """The same document written one value at a time through `Builder` (key vectors shared per key set, element structs
    interleaved with their vectors): a differently laid out but equivalent FlexBuffer, used to exercise the generic reader."""
    b = Builder()
    planes = {}
    for key, attr, fields in _cloud_planes(cloud):
        arr = np.ascontiguousarray(getattr(cloud, attr), np.float32)
        elems = []
        for row in arr:
            m = {}
            for fkey, c0, w in fields:
                m[fkey] = ("f", float(row[c0])) if w == 1 else ("o",) + b.float_vector(row[c0:c0 + w])
            elems.append(("o",) + b.map(m))
        planes[key] = ("o",) + b.vector(elems)
    return b.finish(*b.map(planes))


def encode_gcloud(cloud: PlanarGaussian3d) -> bytes:
    """`PlanarGaussian3d::encode` (src/io/gcloud/flexbuffers.rs:9-16)."""
    b = Builder()
    planes = {}
    for key, attr, fields in _cloud_planes(cloud):
        planes[key] = _encode_plane(b, np.ascontiguousarray(getattr(cloud, attr), np.float32), fields)
    return b.finish(*b.map(planes))


def _decode_plane_fast(pr: "Ref", fields, width: int):
    """Vectorised read of a plane whose N elements are maps with one shared key order, 4-byte slots and 4-byte-aligned
    f32 payloads (what encode_gcloud writes; a regular writer's output in general).  None = not that shape: the caller
    falls back to the generic per-element reader."""
    buf = pr.buf
    if pr.type != FBT_VECTOR or pr.byte_width != 4:
        return None
    t, n, _ = pr._vector_info()
    if n == 0:
        return np.zeros((0, width), np.float32)
    if t % 4 or t + 5 * n > len(buf):
        return None
    u32 = np.frombuffer(buf, "<u4", len(buf) // 4)
    f32 = np.frombuffer(buf, "<f4", len(buf) // 4)
    types = np.frombuffer(buf, np.uint8, n, t + 4 * n)
    if not np.all(types == ((FBT_MAP << 2) | 2)):
        return None
    idx = np.arange(n, dtype=np.int64)
    vals = t + 4 * idx - u32[t // 4: t // 4 + n].astype(np.int64)      # first value slot of every map
    if vals.min() < 12 or np.any(vals % 4):
        return None
    first = pr[0]
    keys = first.keys()
    k = len(keys)
    if np.any(u32[vals // 4 - 1] != k) or np.any(u32[vals // 4 - 2] != 4) or vals.max() + 5 * k > len(buf):
        return None
    kvec = vals - 12 - u32[vals // 4 - 3].astype(np.int64)
    if np.any(kvec != kvec[0]):                                        # one shared key vector <=> one key order
        return None
    arr = np.zeros((n, width), np.float32)
    tbytes = np.frombuffer(buf, np.uint8)
    for fk, c0, w in fields:
        if fk not in keys:
            continue                                                   # #[serde(default)]
        j = keys.index(fk)
        ty = tbytes[vals + 4 * k + j]
        if np.any(ty != ty[0]):
            return None
        slot = vals + 4 * j
        packed = int(ty[0])
        if w == 1:
            if packed != ((FBT_FLOAT << 2) | 2):
                return None
            arr[:, c0] = f32[slot // 4]
            continue
        vty, bw = packed >> 2, 1 << (packed & 3)
        fixed = FBT_VECTOR_INT2 <= vty <= FBT_VECTOR_FLOAT4 and (vty - FBT_VECTOR_INT2) % 3 == FBT_FLOAT - FBT_INT
        if bw != 4 or not (vty == FBT_VECTOR_FLOAT or fixed):
            return None
        tgt = slot - u32[slot // 4].astype(np.int64)
        if tgt.min() < (0 if fixed else 4) or np.any(tgt % 4) or tgt.max() + 4 * w > len(buf):
            return None
        if fixed:
            if (vty - FBT_VECTOR_INT2) // 3 + 2 != w:
                raise FlexBufferError(f"{fk.decode()} has {(vty - FBT_VECTOR_INT2) // 3 + 2} elements, expected {w}")
        elif np.any(u32[tgt // 4 - 1] != w):
            raise FlexBufferError(f"{fk.decode()} does not have {w} elements")
        arr[:, c0:c0 + w] = f32[(tgt // 4)[:, None] + np.arange(w)]
    return arr


def decode_gcloud(data) -> PlanarGaussian3d:
    """`PlanarGaussian3d::decode` (src/io/gcloud/flexbuffers.rs:18-21): structural, like serde -- structs from maps
    (or from sequences in field order), arrays from any vector of numbers; a missing plane is an error, a missing
    FIELD takes its default (`#[serde(default)]`, planar_3d.rs:45-54)."""
    try:
        return _decode_gcloud(data)
    except (KeyError, IndexError, OverflowError, MemoryError) as e:
        raise FlexBufferError(f"malformed gcloud: {type(e).__name__}: {e}") from e


def _decode_gcloud(data) -> PlanarGaussian3d:
    r = root(data)
    if r.type == FBT_MAP:
        top = r.as_dict()
        plane_refs = [top.get(key) for key, _, _ in _PLANES]
    elif r.is_vector() and len(r) >= 4:
        plane_refs = [r[i] for i in range(4)]
    else:
        raise FlexBufferError("a .gcloud root is the PlanarGaussian3d struct (map or 4-sequence)")
    out = []
    n_ref = None
    for (key, _, fields), pr in zip(_PLANES, plane_refs):
        if pr is None or not pr.is_vector():
            raise FlexBufferError(f"plane {key.decode()} missing")
        n = len(pr)
        if n > len(data):
            raise FlexBufferError("element count exceeds the buffer")     # a corrupted length must not size an allocation
        n_ref = n if n_ref is None else n_ref
        if n != n_ref:
            raise FlexBufferError("planes differ in length")
        if key == b"spherical_harmonic":   # the degree the file was written at, from its tuple length
            fields = _sh_fields(_sh_width(pr))
        width = sum(w for _, _, w in fields)
        arr = _decode_plane_fast(pr, fields, width)
        if arr is None:
            arr = _decode_plane_generic(pr, fields, width, n)
        out.append(arr)
    return PlanarGaussian3d(out[0], out[1], out[2], out[3])


def _decode_plane_generic(pr: "Ref", fields, width: int, n: int) -> np.ndarray:
    arr = np.zeros((n, width), np.float32)
    for i in range(n):
        e = pr[i]
        if e.type == FBT_MAP:
            d = e.as_dict()
            vals = [d.get(fk) for fk, _, _ in fields]
        elif e.is_vector():
            vals = [e[j] if j < len(e) else None for j in range(len(fields))]
        else:
            raise FlexBufferError("plane element is not a struct")
        for (fk, c0, w), v in zip(fields, vals):
            if v is None:
                continue
            if w == 1:
                arr[i, c0] = v.as_float()
            else:
                a = v.as_float_array()
                if len(a) != w:
                    raise FlexBufferError(f"{fk.decode()} has {len(a)} elements, expected {w}")
                arr[i, c0:c0 + w] = a
    return arr


def write_gcloud(path, cloud: PlanarGaussian3d) -> None:
    """`CloudCodec::write_to_file` (src/io/codec.rs:8-17)."""
    with open(path, "wb") as f:
        f.write(encode_gcloud(cloud))


def read_gcloud(path) -> PlanarGaussian3d:
    with open(path, "rb") as f:
        return decode_gcloud(f.read())
