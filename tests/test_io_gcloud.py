"""`.gcloud` codec (row f1): the reference pins this format only through a round trip (tests/io.rs:7-17,
tests/gaussian.rs:7-17: decode(encode(random_gaussians_3d(n))) == original) -- restated here -- plus the generic
FlexBuffers reader against buffers assembled by hand from the published wire format (every width, typed / fixed /
untyped vectors, maps, indirect scalars).  Parity with bytes written by the Rust `flexbuffers` crate: unpinned."""
import struct

import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
from bevy_gaussian_splatting_b200 import gcloud as G


def _same(a, b):
    return all(np.array_equal(getattr(a, k).view(np.uint32), getattr(b, k).view(np.uint32))
               for k in ("position_visibility", "spherical_harmonic", "rotation", "scale_opacity"))


@pytest.mark.parametrize("n", [100, 10000])          # the counts of tests/gaussian.rs and tests/io.rs
def test_codec_3d_round_trip(n, tmp_path):
    cloud = B.random_gaussians_3d_seeded(n, 7)
    cloud.scale_opacity[0] = [np.float32(1e-38), -0.0, np.inf, np.float32(3e38)]     # bit patterns survive
    data = G.encode_gcloud(cloud)
    assert _same(G.decode_gcloud(data), cloud)
    p = tmp_path / "c.gcloud"
    G.write_gcloud(p, cloud)
    assert _same(G.read_gcloud(p), cloud) and p.stat().st_size == len(data)
    r = G.root(data)
    assert r.type == G.FBT_MAP and r.keys() == [b"position_visibility", b"rotation", b"scale_opacity", b"spherical_harmonic"]
    e0 = r.as_dict()[b"position_visibility"][0]
    assert e0.type == G.FBT_MAP and e0.keys() == [b"position", b"visibility"]
    assert e0.as_dict()[b"position"].type == G.FBT_VECTOR_INT2 + 3 + 2      # VECTOR_FLOAT3


def test_empty_cloud_and_errors():
    empty = B.PlanarGaussian3d(np.zeros((0, 4), np.float32), np.zeros((0, 48), np.float32), np.zeros((0, 4), np.float32),
                               np.zeros((0, 4), np.float32))
    assert len(G.decode_gcloud(G.encode_gcloud(empty))) == 0
    data = G.encode_gcloud(B.random_gaussians_3d_seeded(3, 1))
    with pytest.raises(G.FlexBufferError):
        G.decode_gcloud(data[:2])
    with pytest.raises(G.FlexBufferError):
        G.decode_gcloud(b"\x00" * 16 + data[-6:])       # root offset points outside / at garbage
    with pytest.raises(G.FlexBufferError):
        G.decode_gcloud(bytes([3, 1, 2, 3, 3, 44, 1]))  # a valid FlexBuffer that is not a cloud


def test_reader_on_hand_assembled_buffers():
    # typed int vector [1, 2, 3], 8-bit: len, elements, root offset, (VECTOR_INT << 2 | 0), root width
    r = G.root(bytes([3, 1, 2, 3, 3, 44, 1]))
    assert r.type == G.FBT_VECTOR_INT and len(r) == 3 and [r[i].as_int() for i in range(3)] == [1, 2, 3]
    assert np.array_equal(r.as_float_array(), np.array([1, 2, 3], np.float32))
    # map { bar: 14, foo: 13 }: keys, key vector (len, offsets), map header (key-vector offset, key width, len), values, types
    buf = b"bar\0foo\0" + bytes([2, 9, 6, 2, 1, 2, 14, 13, 4, 4, 4, 36, 1])
    m = G.root(buf)
    assert m.type == G.FBT_MAP and m.keys() == [b"bar", b"foo"]
    assert {k: v.as_int() for k, v in m.as_dict().items()} == {b"bar": 14, b"foo": 13}
    # untyped vector [f32 1.5 (inline), -> f64 2.25 (indirect), -> VECTOR_FLOAT (16-bit wide? no: 4-byte) of 5 floats], 4-byte slots
    out = bytearray()
    out += struct.pack("<d", 2.25)                                   # indirect f64 at 0
    out += struct.pack("<I", 5); v5 = len(out); out += np.arange(5, dtype="<f4").tobytes()
    out += struct.pack("<I", 3); vec = len(out)
    out += struct.pack("<f", 1.5)
    out += struct.pack("<I", len(out) - 0)
    out += struct.pack("<I", len(out) - v5)
    out += bytes([(G.FBT_FLOAT << 2) | 2, (G.FBT_INDIRECT_FLOAT << 2) | 3, (G.FBT_VECTOR_FLOAT << 2) | 2])
    out += b"\0"                                                     # align the root slot
    out += struct.pack("<I", len(out) - vec) + bytes([(G.FBT_VECTOR << 2) | 2, 4])
    r = G.root(bytes(out))
    assert len(r) == 3 and r[0].as_float() == 1.5 and r[1].as_float() == 2.25
    assert np.array_equal(r[2].as_float_array(), np.arange(5, dtype=np.float32))
    # a cloud whose structs are SEQUENCES (serde also accepts a struct as a tuple) and whose floats are f64 / 16-bit offsets
    b = bytearray()

    def f64vec(vals):
        b.extend(b"\0" * (-len(b) % 8)); b.extend(struct.pack("<Q", len(vals))); p = len(b)
        b.extend(np.asarray(vals, "<f8").tobytes()); return p

    def seq(items):   # items: (position, packed) -> untyped vector with 2-byte slots
        b.extend(b"\0" * (-len(b) % 2)); b.extend(struct.pack("<H", len(items))); p = len(b)
        for pos, _ in items:
            b.extend(struct.pack("<H", len(b) - pos))
        b.extend(bytes(pk for _, pk in items)); return p

    F8 = (G.FBT_VECTOR_FLOAT << 2) | 3
    V2 = (G.FBT_VECTOR << 2) | 1
    b.extend(b"\0" * (-len(b) % 8)); vis_pos = len(b); b.extend(struct.pack("<d", 0.75))    # indirect f64 scalar
    IF8 = (G.FBT_INDIRECT_FLOAT << 2) | 3
    pv = seq([(seq([(f64vec([1, 2, 3]), F8), (vis_pos, IF8)]), V2)])
    sh = seq([(seq([(f64vec(np.arange(48)), F8)]), V2)])
    ro = seq([(seq([(f64vec([1, 0, 0, 0]), F8)]), V2)])
    so = seq([(seq([(f64vec([.5, .25, .125]), F8)]), V2)])                          # opacity missing -> default 0
    top = seq([(pv, V2), (sh, V2), (ro, V2), (so, V2)])
    b.extend(b"\0" * (-len(b) % 2)); b.extend(struct.pack("<H", len(b) - top)); b.extend(bytes([V2, 2]))
    c = G.decode_gcloud(bytes(b))
    assert len(c) == 1 and c.position_visibility.tolist() == [[1, 2, 3, 0.75]] and c.rotation.tolist() == [[1, 0, 0, 0]]
    assert c.scale_opacity.tolist() == [[.5, .25, .125, 0.0]] and np.array_equal(c.spherical_harmonic[0], np.arange(48, dtype=np.float32))


def test_loader_switches_on_the_extension(tmp_path):
    """src/io/loader.rs:38-66: .ply / .gcloud by extension, anything else is an error."""
    from bevy_gaussian_splatting_b200.io import write_ply_3d

    cloud = B.random_gaussians_3d_seeded(64, 2)
    G.write_gcloud(tmp_path / "a.gcloud", cloud)
    assert _same(B.load_cloud(tmp_path / "a.gcloud"), cloud)
    write_ply_3d(tmp_path / "a.ply", cloud)
    assert len(B.load_cloud(tmp_path / "a.ply")) == 64 + 32          # ply.rs:127-129 pads by 32 - n % 32
    with pytest.raises(ValueError):
        B.load_cloud(tmp_path / "a.splat")


def test_fast_and_generic_paths_agree(monkeypatch):
    """encode_gcloud writes every plane with numpy and decode_gcloud reads such regular planes with numpy; documents laid
    out differently (here: written value by value, every struct next to its vectors) go through the generic reader.
    Both must give the same cloud, and a scene-sized cloud must not take minutes."""
    import time

    cloud = B.random_gaussians_3d_seeded(3000, 11)
    fast, slow = G.encode_gcloud(cloud), G.encode_gcloud_elementwise(cloud)
    assert fast != slow and _same(G.decode_gcloud(slow), cloud)
    called = {"generic": 0}
    orig = G._decode_plane_generic
    monkeypatch.setattr(G, "_decode_plane_generic", lambda *a: (called.__setitem__("generic", called["generic"] + 1), orig(*a))[1])
    # both layouts are regular (uniform slots, one key order): the vectorised reader takes all planes of both
    assert _same(G.decode_gcloud(fast), cloud) and _same(G.decode_gcloud(slow), cloud) and called["generic"] == 0
    # and with the vectorised reader switched off the generic one gives the same cloud from both
    monkeypatch.setattr(G, "_decode_plane_fast", lambda *a: None)
    assert _same(G.decode_gcloud(fast), cloud) and _same(G.decode_gcloud(slow), cloud) and called["generic"] == 8
    monkeypatch.undo()
    big = B.random_gaussians_3d_seeded(300_000, 12)
    t0 = time.time()
    data = G.encode_gcloud(big)
    back = G.decode_gcloud(data)
    assert _same(back, big) and time.time() - t0 < 30.0


def test_committed_fixture():
    """tests/golden/c64_seed5.gcloud (written by tests/golden/make_golden.py::make_gcloud_fixture) freezes the codec:
    the reader returns the seeded cloud bit for bit, and the writer still produces the same bytes."""
    import os

    path = os.path.join(os.path.dirname(__file__), "golden", "c64_seed5.gcloud")
    cloud = B.random_gaussians_3d_seeded(64, 5)
    assert _same(G.read_gcloud(path), cloud)
    assert G.encode_gcloud(cloud) == open(path, "rb").read()


def test_cpp_gcloud_reader_and_writer_interoperate_with_python(tmp_path):
    """Row f1: the C++ host mirror (include/bgs_io.hpp: generic FlexBuffers reader, `decode_gcloud` / `encode_gcloud` /
    `load_cloud`) reads what the Python mirror writes -- including the committed golden fixture -- and the other way round."""
    import os
    import subprocess

    import numpy as np
    import bevy_gaussian_splatting_b200 as B

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    subprocess.run(["make", "-C", os.path.join(root, "examples"), "-s", "cloud_tool"], check=True)
    tool = os.path.join(root, "examples", "cloud_tool")

    def planes(path):
        raw = open(path, "rb").read()
        n = int(np.frombuffer(raw, "<u8", 1)[0])
        off, out = 8, []
        for w in (4, 48, 4, 4):
            out.append(np.frombuffer(raw, "<f4", n * w, off).reshape(n, w)); off += n * w * 4
        return out

    cloud = B.random_gaussians_3d_seeded(1237, 9)
    cloud.position_visibility[5, 0] = np.float32("nan"); cloud.scale_opacity[7, 3] = np.float32("inf")
    B.write_gcloud(tmp_path / "py.gcloud", cloud)
    for src in (tmp_path / "py.gcloud", *[os.path.join(root, "tests", "golden", f) for f in sorted(os.listdir(os.path.join(root, "tests", "golden"))) if f.endswith(".gcloud")]):
        want = B.read_gcloud(src)
        r = subprocess.run([tool, str(src), str(tmp_path / "out.bin")], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        got = planes(tmp_path / "out.bin")
        for g, w in zip(got, (want.position_visibility, want.spherical_harmonic, want.rotation, want.scale_opacity)):
            assert np.array_equal(g.view(np.uint32), w.view(np.uint32))
    # C++ writer -> Python reader (and -> C++ reader again)
    r = subprocess.run([tool, str(tmp_path / "py.gcloud"), str(tmp_path / "cpp.gcloud"), "--gcloud"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    back = B.read_gcloud(tmp_path / "cpp.gcloud")
    for a, b in ((back.position_visibility, cloud.position_visibility), (back.spherical_harmonic, cloud.spherical_harmonic),
                 (back.rotation, cloud.rotation), (back.scale_opacity, cloud.scale_opacity)):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    subprocess.run([tool, str(tmp_path / "cpp.gcloud"), str(tmp_path / "out2.bin")], check=True, capture_output=True)
    assert all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(planes(tmp_path / "out2.bin"), planes(tmp_path / "out.bin") if False else
               [cloud.position_visibility, cloud.spherical_harmonic, cloud.rotation, cloud.scale_opacity]))
    # malformed input: a status, not a crash
    (tmp_path / "bad.gcloud").write_bytes(open(tmp_path / "py.gcloud", "rb").read()[:-7])
    assert subprocess.run([tool, str(tmp_path / "bad.gcloud"), str(tmp_path / "o.bin")], capture_output=True).returncode == 2


def test_damaged_files_are_errors_in_both_hosts(tmp_path):
    """Truncated, bit-flipped and tail-corrupted `.ply` / `.gcloud` files: the Python loaders raise ValueError, the C++ loader
    exits with its error code -- never a crash, a hang or an allocation sized by a corrupted count (the loaders of the
    reference return io::Error, src/io/loader.rs:38-66)."""
    import io as pyio
    import os
    import subprocess

    import bevy_gaussian_splatting_b200.io as IO

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    subprocess.run(["make", "-C", os.path.join(root, "examples"), "-s", "cloud_tool"], check=True)
    tool = os.path.join(root, "examples", "cloud_tool")
    cloud = B.random_gaussians_3d_seeded(29, 3)
    IO.write_ply_3d(tmp_path / "a.ply", cloud)
    G.write_gcloud(tmp_path / "a.gcloud", cloud)
    rng = np.random.default_rng(11)
    outcomes = set()
    for ext in ("ply", "gcloud"):
        data = (tmp_path / f"a.{ext}").read_bytes()
        for it in range(40):
            b = bytearray(data)
            mode = it % 3
            if mode == 0:
                b = b[: int(rng.integers(0, len(b)))]
            elif mode == 1:
                for _ in range(int(rng.integers(1, 8))):
                    b[int(rng.integers(0, len(b)))] = int(rng.integers(0, 256))
            else:   # the flexbuffer root and the plane offsets live at the END of a .gcloud; the header at the start of a .ply
                lo = max(0, len(b) - 64) if ext == "gcloud" else 0
                for _ in range(int(rng.integers(1, 6))):
                    b[lo + int(rng.integers(0, 64))] = int(rng.integers(0, 256))
            try:
                if ext == "ply":
                    IO.parse_ply_3d(pyio.BytesIO(bytes(b)))
                else:
                    G.decode_gcloud(bytes(b))
                outcomes.add((ext, "py-ok"))
            except ValueError:
                outcomes.add((ext, "py-error"))
            if it % 4 == 0:   # (a process per case: a sample is enough here)
                fn = tmp_path / f"m.{ext}"
                fn.write_bytes(bytes(b))
                r = subprocess.run([tool, str(fn), str(tmp_path / "o.bin")], capture_output=True, timeout=60)
                assert r.returncode in (0, 2), (ext, it, r.returncode, r.stderr.decode()[-300:])
                outcomes.add((ext, "cpp-ok" if r.returncode == 0 else "cpp-error"))
    assert {("ply", "py-error"), ("gcloud", "py-error"), ("ply", "cpp-error"), ("gcloud", "cpp-error")} <= outcomes
    # the one the sanitizer run found: a plane whose length slot claims more elements than the buffer has bytes
    with pytest.raises(ValueError):
        bad = bytearray((tmp_path / "a.gcloud").read_bytes())
        G.decode_gcloud(bytes(bad[:-3]) + b"\xff\xff\xff")
