"""RasterizeMode::Classification and RasterizeMode::OpticalFlow on the CPU: the oracle's colour sources
(modes_oracle/) against the independent numpy restatement in `modes_cases`, bit for bit, on inputs built to reach each
branch; the restated hsv_to_rgb against Python's colorsys (Bevy is not available, so this pins the formula); the fixed
atan2 series against numpy's; and the C header's new struct and call from a C99 program."""
import colorsys
import ctypes as C
import os
import subprocess
import textwrap

import numpy as np
import pytest

import modes_cases as MC
from bevy_gaussian_splatting_b200 import abi
from modes_oracle import modes_oracle as MO

f32 = np.float32
U = 2.0 ** -24


def assert_same_bits(got, want, what):
    ok = MC.same_bits(got, want)
    if not ok.all():
        i = np.argwhere(~ok)[0]
        raise AssertionError(f"{what}: first difference at {tuple(i)}: {got[tuple(i)]!r} vs {want[tuple(i)]!r}")


def test_hsv_to_rgb_matches_colorsys_inside_each_sextant():
    """|restated - colorsys| <= 32 U: h / FRAC_PI_3 carries U plus FRAC_PI_3's own rounding (0.47 U relative) on |h / F| <= 6,
    x = base + hk a further U on |x| <= 11, the remainder's steps U each on |k| < 6 (6 * trunc and the difference are exact
    for |x| < 12): k is within 6 (1.47 U) + 11 U + 6 U < 26 U; v - (v s) m adds 3 U on values <= 1.  32 U covers it."""
    rng = np.random.default_rng(0)
    for sx in range(6):
        lo, hi = sx * np.pi / 3, (sx + 1) * np.pi / 3
        h = rng.uniform(lo + 1e-4, hi - 1e-4, 400).astype(f32)
        s, v = rng.uniform(0, 1, 400).astype(f32), rng.uniform(0, 1, 400).astype(f32)
        got = MC.hsv_to_rgb(h, s, v).astype(np.float64)
        want = np.array([colorsys.hsv_to_rgb(float(a) / (2 * np.pi), float(b), float(c)) for a, b, c in zip(h, s, v)])
        err = np.abs(got - want).max()
        assert err <= 32 * U, f"sextant {sx}: {err:.3g}"


@pytest.mark.parametrize("num_classes", MC.NUM_CLASSES)
def test_class_colour_bit_exact(num_classes):
    vis = MC.class_labels(num_classes)
    rng = np.random.default_rng(num_classes)
    sh = rng.uniform(-0.2, 1.3, (len(vis), 3)).astype(f32)
    sh[:4] = [[0, 0, 0], [1, 1, 1], [-0.0, 0.5, 1e-38], [3e38, -3e38, 1e-45]]
    want = MC.class_colour(sh, vis, num_classes)
    assert_same_bits(MO.class_colour(sh, vis, num_classes), want, f"class colour, num_classes {num_classes}")
    below = vis < 2
    assert_same_bits(want[below], sh[below], "vis < 2 keeps the sh colour")
    assert not MC.same_bits(want[~below], sh[~below]).all(axis=1).any()
    # the pool tells WGSL's remainder from fmodf's (a mutant the bit-exact checks must see)
    hue = ((vis - f32(2)) / f32(num_classes)) * MC.TAU_CLASS
    with np.errstate(all="ignore"):
        x = f32(5) + hue / MC.FRAC_PI_3
        k_fmod = np.fmod(x, f32(6))
        alt = f32(1) - np.fmax(f32(0), np.fmin(k_fmod, np.fmin(f32(4) - k_fmod, f32(1))))
    assert (~MC.same_bits(alt, MC.hsv_to_rgb(hue, f32(1), f32(1))[:, 0]) & (vis >= 2)).any()
    # one hue per whole class: 2 + k and 2 + k + num_classes agree only up to the wrap's rounding, classes differ
    if num_classes == 3:
        h = MC.class_colour(np.zeros((3, 3), f32), f32(2) + np.arange(3, dtype=f32), 3)
        assert len({tuple(r) for r in h.tolist()}) == 3


def test_hsv_to_rgb_bit_exact_on_specials():
    h = np.concatenate([np.array([0, -0.0, np.pi, -np.pi, 2 * np.pi, 1e30, -1e30, np.inf, -np.inf, np.nan, 1e-45], f32),
                        np.arange(-20, 40, dtype=f32) * f32(np.pi / 3), np.nextafter(np.arange(7, dtype=f32) * f32(np.pi / 3), f32(9))])
    for s in (0.0, 0.5, 1.0, np.nan):
        assert_same_bits(MO.hsv_to_rgb(h, f32(s), f32(1)), MC.hsv_to_rgb(h, f32(s), f32(1)), f"hsv_to_rgb s={s}")


def test_atan2_series_bit_exact_and_accurate():
    fl = MC.sextant_flows()
    rng = np.random.default_rng(1)
    y = np.concatenate([fl[:, 1], rng.normal(0, 1, 5000).astype(f32), (rng.normal(0, 1, 2000) * 1e-30).astype(f32)])
    x = np.concatenate([fl[:, 0], rng.normal(0, 1, 5000).astype(f32), (rng.normal(0, 1, 2000) * 1e30).astype(f32)])
    got = MO.atan2(y, x)
    assert_same_bits(got, MC.atan2(y, x), "atan2")
    want = np.arctan2(y.astype(np.float64), x.astype(np.float64))
    fin = np.isfinite(want)
    ulp = np.spacing(np.abs(want[fin]).astype(f32)).astype(np.float64)
    assert (np.abs(got[fin] - want[fin]) <= ulp).all(), "the series is more than 1 ulp from atan2"
    # the exact values the rule depends on
    pi = f32(np.pi)
    sp = MO.atan2(np.array([0.0, -0.0, 0.0, -0.0, 0.0], f32), np.array([1.0, 1.0, -1.0, -1.0, 0.0], f32))
    assert_same_bits(sp, np.array([0.0, -0.0, pi, -pi, 0.0], f32), "atan2 at +-0 and +-pi")
    assert f32(-pi) + MC.PI_2 == pi            # + PI_2 turns -pi into pi exactly


def test_flow_colour_bit_exact_each_sextant():
    pv = np.array([[0, 0, 0, 1]], f32)
    eye = np.eye(4, dtype=f32).reshape(-1)
    seen = set()
    for fx, fy in MC.sextant_flows():
        prev = MC.translated(fx, fy)
        got = MO.flow_colour(pv, eye, eye, prev, 1.0)
        assert_same_bits(got, MC.flow_colour(pv, eye, eye, prev, 1.0), f"flow ({fx}, {fy})")
        if np.isfinite([fx, fy]).all() and (fx, fy) != (0, 0):
            ang = np.arctan2(-0.0 if fy == 0 else fy, fx) % (2 * np.pi)
            seen.add(int(ang // (np.pi / 3)) % 6)
            r = np.hypot(fx, fy)
            want = colorsys.hsv_to_rgb(ang / (2 * np.pi), min(r, 1.0), 1.0)
            assert np.abs(got[0] - want).max() <= 32 * U + 1e-6, (fx, fy, got, want)
    assert seen == set(range(6))
    # zero motion: atan2(0, 0) = 0 and saturation 0 -> white
    assert_same_bits(MO.flow_colour(pv, eye, eye, eye, 1.0), np.ones((1, 3), f32), "zero motion")


def test_flow_colour_bit_exact_moving_camera():
    cur, prevs, rng = MC.camera_matrices(0)
    pos = np.concatenate([rng.uniform(-3, 3, (3000, 3)), rng.uniform(-1e3, 1e3, (200, 3)), np.zeros((2, 3))]).astype(f32)
    pv = np.concatenate([pos, np.ones((len(pos), 1), f32)], 1)
    model = np.array([[0.5, 0.1, 0, 1], [0, 1, 0.2, -1], [0, 0, 2, 0.5], [0, 0, 0, 1]], f32)
    for mname, m in (("identity", np.eye(4, dtype=f32)), ("affine", model)):
        mt = np.ascontiguousarray(m.T).reshape(-1)
        for name, prev in prevs.items():
            for dt in (1 / 60, 0.5, 1e-6):
                want = MC.flow_colour(pv, mt, cur, prev, dt)
                assert_same_bits(MO.flow_colour(pv, mt, cur, prev, dt), want, f"{mname} {name} dt={dt}")
                if name == "still":
                    assert_same_bits(want, np.ones_like(want), "still camera -> white")
    # a previous w <= 0 (a point behind the previous camera) takes the non-finite path on both sides alike
    c = MC.mat4_point(prevs["behind"], pos)
    assert (c[:, 3] <= 0).any()


def test_extras_struct_and_call_compile_as_c99(tmp_path):
    assert C.sizeof(abi.bgs_render_extras) == 72
    assert [n for n, _, _ in abi.SYMBOLS].count("bgs_render_ex") == 1
    root = os.path.join(os.path.dirname(__file__), "..")
    src = tmp_path / "ex.c"
    src.write_text(textwrap.dedent("""
        #include <stdio.h>
        #include "bgs.h"
        int main(void) {
            bgs_render_extras ex = {{1,0,0,0, 0,1,0,0, 0,0,1,0, 0,0,0,1}, 1.0f / 60.0f, 3u};
            bgs_settings s = {BGS_GAUSSIAN_3D, BGS_RASTERIZE_CLASSIFICATION, 0, 1, BGS_DRAW_ALL, 32, 0, 0};
            bgs_status st = bgs_render_ex(NULL, NULL, NULL, NULL, &s, &ex, NULL, BGS_FORMAT_RGBA32F, 0);
            printf("%d %u %d\\n", (int)st, (unsigned)sizeof(ex), (int)BGS_RASTERIZE_OPTICAL_FLOW);
            return 0;
        }
    """))
    exe = tmp_path / "ex"
    libdir = os.path.join(root, "bevy_gaussian_splatting_b200")
    subprocess.run(["/usr/bin/gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(root, "include"), str(src),
                    "-o", str(exe), "-L", libdir, "-lbgs", f"-Wl,-rpath,{libdir}"], check=True, capture_output=True, text=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()
    assert out == [str(abi.BGS_EINVAL), "72", "5"]
