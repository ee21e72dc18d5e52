"""Clouds at SH degree 0, 1 and 2 on the host, without a GPU: the ply f_rest_ rule of an sh_d build (quirks included),
ply and .gcloud round trips at every width between the Python and C++ hosts, f16 packing at every width, the oracle's
colour of a zero-padded degree-d cloud against the numpy restatement of the degree-d colour, and the new ABI calls."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
import sh_degree_cases as SC
from bevy_gaussian_splatting_b200 import abi
from bevy_gaussian_splatting_b200.gaussian import SH_WIDTHS, sh_degree_of_width
from bevy_gaussian_splatting_b200.io import parse_ply_3d, write_ply_3d

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ALL_DEGREES = (0, 1, 2, 3)


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.fixture(scope="module")
def cloud_tool():
    subprocess.run(["make", "-C", os.path.join(ROOT, "examples"), "-s", "cloud_tool"], check=True)
    return os.path.join(ROOT, "examples", "cloud_tool")


def dumped_planes(path, d):
    raw = open(path, "rb").read()
    n = int(np.frombuffer(raw, "<u8", 1)[0])
    off, out = 8, []
    for w in (4, SH_WIDTHS[d], 4, 4):
        out.append(np.frombuffer(raw, "<f4", n * w, off).reshape(n, w)); off += n * w * 4
    assert off == len(raw)
    return out


def ply_with_rest(path, n_rest: int, n: int = 5) -> np.ndarray:
    """A ply whose f_rest_i of gaussian j is 1000 j + i + 1 (so a value names its property); returns those values."""
    props = ["x", "y", "z", "f_dc_0", "f_dc_1", "f_dc_2"] + [f"f_rest_{i}" for i in range(n_rest)] + \
            ["opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"]
    arr = np.zeros(n, np.dtype([(p, "<f4") for p in props]))
    rest = np.array([[1000 * j + i + 1 for i in range(n_rest)] for j in range(n)], np.float32).reshape(n, n_rest)
    for i in range(n_rest):
        arr[f"f_rest_{i}"] = rest[:, i]
    for c in range(3):
        arr[f"f_dc_{c}"] = -1.0 - c
    arr["rot_0"] = 1.0
    with open(path, "wb") as f:
        f.write(("ply\nformat binary_little_endian 1.0\nelement vertex %d\n" % n).encode())
        for p in props:
            f.write(f"property float {p}\n".encode())
        f.write(b"end_header\n")
        f.write(arr.tobytes())
    return rest


# ---- the plane width and the degree


@pytest.mark.parametrize("width", [0, 3, 8, 16, 27, 47, 49, 76])
def test_other_sh_widths_are_refused(width):
    with pytest.raises(ValueError):
        B.PlanarGaussian3d(np.zeros((2, 4)), np.zeros((2, width)), np.zeros((2, 4)), np.zeros((2, 4)))


@pytest.mark.parametrize("d", ALL_DEGREES)
def test_sh_degree_follows_the_width(d):
    c = B.random_gaussians_3d_seeded(100, 4, sh_degree=d)
    assert c.spherical_harmonic.shape == (100, SH_WIDTHS[d]) and c.sh_degree == d == sh_degree_of_width(SH_WIDTHS[d])
    full = B.random_gaussians_3d_seeded(100, 4)
    k = 3 * (d + 1) ** 2
    # the lower bands of the same draws, padding lanes zero; the default stream is untouched
    assert np.array_equal(bits(c.spherical_harmonic[:, :k]), bits(full.spherical_harmonic[:, :k]))
    assert not c.spherical_harmonic[:, k:].any()
    for a, b in ((c.position_visibility, full.position_visibility), (c.rotation, full.rotation),
                 (c.scale_opacity, full.scale_opacity)):
        assert np.array_equal(bits(a), bits(b))
    # with_sh_degree(3) zero-pads; going back down gives the same cloud
    up = c.with_sh_degree(3)
    assert up.sh_degree == 3 and np.array_equal(bits(up.with_sh_degree(d).spherical_harmonic), bits(c.spherical_harmonic))


def test_default_generator_is_unchanged():
    a, b = B.random_gaussians_3d_seeded(3000, 11), B.random_gaussians_3d_seeded(3000, 11, sh_degree=3)
    assert a.sh_degree == 3 and np.array_equal(bits(a.spherical_harmonic), bits(b.spherical_harmonic))


# ---- f16 packing


@pytest.mark.parametrize("d", ALL_DEGREES)
def test_f16_pack_and_decode_at_every_width(d, oracle):
    c = SC.with_padding_noise(B.random_gaussians_3d_seeded(257, 6, sh_degree=d), 6) if d in (0, 2) else \
        B.random_gaussians_3d_seeded(257, 6, sh_degree=d)
    shp, rso = c.pack_f16()
    assert shp.shape == (257, SH_WIDTHS[d] // 2) and shp.dtype == np.uint32
    back = B.PlanarGaussian3d.from_f16(c.position_visibility, shp, rso)
    assert back.sh_degree == d
    assert np.array_equal(bits(back.spherical_harmonic), bits(c.rounded_to_f16().spherical_harmonic))
    assert np.array_equal(back.pack_f16()[0], shp)
    # the oracle's packing of the zero-extended plane holds the same words first, zero words after
    o_shp, o_rso = oracle.pack_f16(SC.embed48(c.spherical_harmonic), c.rotation, c.scale_opacity)
    assert np.array_equal(o_shp, SC.embed24(shp)) and np.array_equal(o_rso, rso)
    with pytest.raises(ValueError):
        B.PlanarGaussian3d.from_f16(c.position_visibility, shp[:, :-1], rso)


# ---- ply


@pytest.mark.parametrize("d", ALL_DEGREES)
def test_ply_rest_placement_follows_the_sh_d_rule(d, tmp_path, cloud_tool):
    """Every f_rest_i of 0..44 lands where the sh_d rule puts it (or nowhere): for sh0, f_rest_0 in padding lane 3 and
    every later one overwriting it (channel i / 1 >= 3 drops all but i = 0); later properties overwrite earlier."""
    rest = ply_with_rest(tmp_path / "r.ply", 45)
    got = parse_ply_3d(tmp_path / "r.ply", sh_degree=d)
    assert got.sh_degree == d
    want = np.zeros((5, SH_WIDTHS[d]), np.float32)
    want[:, :3] = [-1.0, -2.0, -3.0]
    for i in range(45):
        idx = SC.rest_index(i, d)
        if idx is not None:
            want[:, idx] = rest[:, i]
    assert np.array_equal(bits(got.spherical_harmonic[:5]), bits(want))
    if d == 0:
        assert np.array_equal(got.spherical_harmonic[:5, 3], rest[:, 0])      # sh0 keeps f_rest_0 in padding lane 3
    if d == 3:
        assert np.array_equal(bits(got.spherical_harmonic), bits(parse_ply_3d(tmp_path / "r.ply").spherical_harmonic))
    # the C++ reader applies the same rule
    r = subprocess.run([cloud_tool, str(tmp_path / "r.ply"), str(tmp_path / "r.bin"), "--sh-degree", str(d)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    for a, b in zip(dumped_planes(tmp_path / "r.bin", d), (got.position_visibility, got.spherical_harmonic, got.rotation,
                                                           got.scale_opacity)):
        assert np.array_equal(a.view(np.uint32), bits(b))


@pytest.mark.parametrize("d", ALL_DEGREES)
def test_ply_writer_round_trip(d, tmp_path, cloud_tool):
    c = B.random_gaussians_3d_seeded(96, 8, sh_degree=d)
    write_ply_3d(tmp_path / "c.ply", c)
    header = open(tmp_path / "c.ply", "rb").read().split(b"end_header")[0].decode()
    assert len(re.findall(r"property float f_rest_\d+", header)) == 3 * ((d + 1) ** 2 - 1)
    back = parse_ply_3d(tmp_path / "c.ply", sh_degree=d)
    # what the file holds, placed by the reader's rule (channel-major writer, i / K_d reader: the reference's quirk)
    rest = (d + 1) ** 2 - 1
    want = np.zeros_like(c.spherical_harmonic)
    want[:, :3] = c.spherical_harmonic[:, :3]
    for i in range(3 * rest):
        idx = SC.rest_index(i, d)
        if idx is not None:
            want[:, idx] = c.spherical_harmonic[:, ((i % rest) + 1) * 3 + i // rest]
    assert np.array_equal(bits(back.spherical_harmonic[:96]), bits(want))
    r = subprocess.run([cloud_tool, str(tmp_path / "c.ply"), str(tmp_path / "c.bin"), "--sh-degree", str(d)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    # (the position and SH planes are copied; exp and the rotation's normalisation may round differently in C++)
    pos, sh, _, _ = dumped_planes(tmp_path / "c.bin", d)
    assert np.array_equal(pos.view(np.uint32), bits(back.position_visibility))
    assert np.array_equal(sh.view(np.uint32), bits(back.spherical_harmonic))


# ---- .gcloud


@pytest.mark.parametrize("d", ALL_DEGREES)
def test_gcloud_round_trip_between_hosts(d, tmp_path, cloud_tool):
    c = B.random_gaussians_3d_seeded(133, 2, sh_degree=d)
    if d in (0, 2):
        c = SC.with_padding_noise(c, 2)    # padding lanes travel with the tuple
    B.write_gcloud(tmp_path / "py.gcloud", c)
    planes = (c.position_visibility, c.spherical_harmonic, c.rotation, c.scale_opacity)
    back = B.read_gcloud(tmp_path / "py.gcloud")
    assert back.sh_degree == d
    assert all(np.array_equal(bits(a), bits(b)) for a, b in
               zip((back.position_visibility, back.spherical_harmonic, back.rotation, back.scale_opacity), planes))
    from bevy_gaussian_splatting_b200.gcloud import decode_gcloud, encode_gcloud_elementwise
    gen = decode_gcloud(encode_gcloud_elementwise(c))    # the generic reader infers the width too
    assert np.array_equal(bits(gen.spherical_harmonic), bits(c.spherical_harmonic))
    # Python -> C++ reader, C++ writer -> Python reader
    r = subprocess.run([cloud_tool, str(tmp_path / "py.gcloud"), str(tmp_path / "py.bin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert all(np.array_equal(a.view(np.uint32), bits(b)) for a, b in zip(dumped_planes(tmp_path / "py.bin", d), planes))
    r = subprocess.run([cloud_tool, str(tmp_path / "py.gcloud"), str(tmp_path / "cpp.gcloud"), "--gcloud"],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    cpp = B.read_gcloud(tmp_path / "cpp.gcloud")
    assert cpp.sh_degree == d and np.array_equal(bits(cpp.spherical_harmonic), bits(c.spherical_harmonic))


def test_gcloud_of_another_sh_width_is_refused(tmp_path, cloud_tool):
    from bevy_gaussian_splatting_b200.gcloud import Builder, FlexBufferError, decode_gcloud

    c = B.random_gaussians_3d_seeded(3, 1)
    b = Builder()
    planes = {}
    widths = {b"position_visibility": None, b"spherical_harmonic": 20, b"rotation": None, b"scale_opacity": None}
    for key, attr in ((b"position_visibility", "position_visibility"), (b"spherical_harmonic", "spherical_harmonic"),
                      (b"rotation", "rotation"), (b"scale_opacity", "scale_opacity")):
        arr = getattr(c, attr)
        elems = []
        for row in arr:
            if key == b"spherical_harmonic":
                m = {b"coefficients": ("o",) + b.float_vector(row[:widths[key]])}
            elif key == b"position_visibility":
                m = {b"position": ("o",) + b.float_vector(row[:3]), b"visibility": ("f", float(row[3]))}
            elif key == b"rotation":
                m = {b"rotation": ("o",) + b.float_vector(row)}
            else:
                m = {b"scale": ("o",) + b.float_vector(row[:3]), b"opacity": ("f", float(row[3]))}
            elems.append(("o",) + b.map(m))
        planes[key] = ("o",) + b.vector(elems)
    data = b.finish(*b.map(planes))
    with pytest.raises(FlexBufferError):
        decode_gcloud(data)
    (tmp_path / "w20.gcloud").write_bytes(data)
    assert subprocess.run([cloud_tool, str(tmp_path / "w20.gcloud"), str(tmp_path / "o.bin")], capture_output=True).returncode == 2


# ---- the colour rule


@pytest.mark.parametrize("d", ALL_DEGREES)
@pytest.mark.parametrize("srgb", [False, True])
def test_oracle_colour_of_the_padded_cloud_is_the_degree_d_colour(d, srgb, oracle):
    """The oracle evaluates 16 bands; on the zero-padded cloud that is the degree-d sum (within the f32 colour
    bound), and non-zero padding lanes of the degree-d cloud do not enter it."""
    view = B.headless_view(320, 240)
    c = SC.with_padding_noise(B.random_gaussians_3d_seeded(4000, 21 + d, sh_degree=d), 5) if d in (0, 2) else \
        B.random_gaussians_3d_seeded(4000, 21 + d, sh_degree=d)
    padded = c.with_sh_degree(3)
    s = B.CloudSettings(global_scale=0.25, color_space=B.GaussianColorSpace(0 if srgb else 1))
    u = B.GaussianSplattingPlugin.cloud_uniform(s, None, padded.compute_aabb())
    rec = oracle.project(padded, view.to_abi(), u, s.to_abi(), np.arange(len(c), dtype=np.uint32))
    drawn = (rec["xlo"] <= rec["xhi"]) & (rec["ylo"] <= rec["yhi"])
    assert drawn.sum() > 100
    want = SC.colour(c, view.world_position, srgb)[drawn]
    got = np.stack([rec["r"], rec["g"], rec["b"]], axis=1)[drawn].astype(np.float64)
    err = np.abs(got - want) / np.maximum(1.0, np.abs(want))
    assert err.max() < 2e-5, err.max()


# ---- the C ABI


NEW_SYMBOLS = {
    "bgs_cloud_upload_f32_sh": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32] + [C.c_void_p] * 4 + [C.POINTER(C.c_void_p)]),
    "bgs_cloud_upload_f16_sh": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32] + [C.c_void_p] * 3 + [C.POINTER(C.c_void_p)]),
    "bgs_cloud_upload_f16_cov_sh": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32] + [C.c_void_p] * 3 + [C.POINTER(C.c_void_p)]),
    "bgs_cloud_download_f32_sh": (C.c_int, [C.c_void_p] * 6),
    "bgs_cloud_download_f16_sh": (C.c_int, [C.c_void_p] * 5),
    "bgs_cloud_sh_degree": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint32)]),
}


def test_new_symbols_are_declared_bound_and_exported():
    lib = abi.load()
    bound = {n: (r, a) for n, r, a in abi.SYMBOLS}
    header = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "bgs.h")).read(), flags=re.S)
    for name, (restype, argtypes) in NEW_SYMBOLS.items():
        assert hasattr(lib, name) and re.search(rf"\b{name}\s*\(", header), name
        assert bound[name][0] == restype and bound[name][1] == argtypes, name
        # the C declaration's parameter count matches the binding's
        decl = re.search(rf"\b{name}\s*\(([^;]*)\)\s*;", header).group(1)
        assert decl.count(",") + 1 == len(argtypes), name
    # the degree sits right after n in every _sh upload
    for name in ("bgs_cloud_upload_f32_sh", "bgs_cloud_upload_f16_sh", "bgs_cloud_upload_f16_cov_sh"):
        decl = re.search(rf"\b{name}\s*\(([^;]*)\)\s*;", header).group(1)
        assert re.match(r"\s*bgs_context\* ctx, uint32_t n, uint32_t sh_degree, const float\* pos_vis,", decl), name


def test_new_calls_refuse_null_arguments_without_a_device():
    lib = abi.load()
    d = C.c_uint32(7)
    assert lib.bgs_cloud_sh_degree(None, C.byref(d)) == abi.BGS_EINVAL and d.value == 7
    assert lib.bgs_cloud_sh_degree(None, None) == abi.BGS_EINVAL
    out = C.c_void_p()
    assert lib.bgs_cloud_upload_f32_sh(None, 1, 0, None, None, None, None, C.byref(out)) == abi.BGS_EINVAL
    assert lib.bgs_cloud_upload_f16_sh(None, 1, 0, None, None, None, C.byref(out)) == abi.BGS_EINVAL
    assert lib.bgs_cloud_upload_f16_cov_sh(None, 1, 0, None, None, None, C.byref(out)) == abi.BGS_EINVAL
    assert not out.value
