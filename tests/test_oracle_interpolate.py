"""The interpolation oracle (interpolate_oracle/) against an independent numpy float32 / float16 transliteration of
src/morph/interpolate.wgsl:51-119 over planar.wgsl's f32 and f16 getters and setters, bit for bit (NaN compared as a
class), on every class of tests/interpolate_cases.py; and that every class is reached."""
import numpy as np
import pytest

import interpolate_cases as IC
from interpolate_oracle import interpolate_oracle as IO

F = np.float32


# ---- the transliteration ------------------------------------------------------------------------------------------
def wgsl_factor(time, time_start, time_stop):
    """interpolate.wgsl:51-57 in f32.  clamp(e, lo, hi) = min(max(e, lo), hi); a -0 quotient is not below 0 and stays."""
    time, time_start, time_stop = F(time), F(time_start), F(time_stop)
    duration = time_stop - time_start
    if abs(duration) < F(1e-6):
        return F(1.0) if time >= time_stop else F(0.0)
    e = (time - time_start) / duration
    e = F(0.0) if e < 0 else e
    return F(1.0) if e > 1 else e


def mix(a, b, t):
    """WGSL mix(e1, e2, e3) = e1 * (1 - e3) + e2 * e3, each operation one f32 rounding."""
    return a * (F(1.0) - t) + b * t


def normalize_quaternion(q):
    """interpolate.wgsl:59-65: dot(q, q) left to right, (0, 0, 0, 1) when it is <= 0."""
    l2 = ((q[:, 0] * q[:, 0] + q[:, 1] * q[:, 1]) + q[:, 2] * q[:, 2]) + q[:, 3] * q[:, 3]
    out = q / np.sqrt(l2)[:, None]
    out[l2 <= 0] = np.array([0, 0, 0, 1], F)
    return out


def unpack2x16float(w):
    """-> (.x = low half, .y = high half) as f32."""
    w = np.asarray(w, np.uint32)
    return ((w & 0xFFFF).astype(np.uint16).view(np.float16).astype(F), (w >> 16).astype(np.uint16).view(np.float16).astype(F))


def pack2x16float(x, y):
    """x -> low half, y -> high half, each rounded to nearest even."""
    lo = np.asarray(x, F).astype(np.float16).view(np.uint16).astype(np.uint32)
    hi = np.asarray(y, F).astype(np.float16).view(np.uint16).astype(np.uint32)
    return (hi << 16) | lo


def wgsl_f32(lhs, rhs, t):
    """PACKED_F32 off, PLANAR_F32 (planar.wgsl:334-430): the lanes are the planes themselves."""
    (pl, shl, rl, sol), (pr, shr, rr, sor) = lhs, rhs
    pos = mix(pl, pr, t)                                                     # position and visibility
    sh = mix(shl, shr, t)
    rot = normalize_quaternion(mix(rl, rr, t))
    so = np.concatenate([mix(sol[:, :3], sor[:, :3], t), mix(sol[:, 3:], sor[:, 3:], t)], axis=1)
    return pos, sh, rot, so


def wgsl_f16(lhs, rhs, t, cov):
    """PLANAR_F16 (planar.wgsl:116-331)."""
    def sh_of(w):                                                            # planar_f16_decode_sh
        lo, hi = unpack2x16float(w)
        out = np.empty((len(w), 48), F)
        out[:, 0::2], out[:, 1::2] = lo, hi
        return out

    (pl, shl, wl), (pr, shr, wr) = lhs, rhs
    pos = mix(pl, pr, t)
    sh = mix(sh_of(shl), sh_of(shr), t)
    sh_out = pack2x16float(sh[:, 0::2], sh[:, 1::2])                          # set_output_spherical_harmonics
    if cov:
        def cov_of(w):                                                       # planar_f16_decode_covariance
            c0, c1, c2 = unpack2x16float(w[:, 0]), unpack2x16float(w[:, 1]), unpack2x16float(w[:, 2])
            return np.stack([c0[1], c0[0], c1[1], c1[0], c2[1], c2[0]], axis=1)
        c = mix(cov_of(wl), cov_of(wr), t)
        op = mix(unpack2x16float(wl[:, 3])[1], unpack2x16float(wr[:, 3])[1], t)
        second = np.stack([pack2x16float(c[:, 1], c[:, 0]), pack2x16float(c[:, 3], c[:, 2]),
                           pack2x16float(c[:, 5], c[:, 4]), pack2x16float(np.zeros_like(op), op)], axis=1)
    else:
        def rot_of(w):                                                       # planar_f16_decode_rotation
            q0, q1 = unpack2x16float(w[:, 0]), unpack2x16float(w[:, 1])
            return np.stack([q0[1], q0[0], q1[1], q1[0]], axis=1)

        def scale_of(w):                                                     # planar_f16_decode_scale
            s0, s1 = unpack2x16float(w[:, 2]), unpack2x16float(w[:, 3])
            return np.stack([s0[1], s0[0], s1[1]], axis=1)

        r = normalize_quaternion(mix(rot_of(wl), rot_of(wr), t))
        s = mix(scale_of(wl), scale_of(wr), t)
        op = mix(unpack2x16float(wl[:, 3])[0], unpack2x16float(wr[:, 3])[0], t)
        second = np.stack([pack2x16float(r[:, 1], r[:, 0]), pack2x16float(r[:, 3], r[:, 2]),
                           pack2x16float(s[:, 1], s[:, 0]), pack2x16float(op, s[:, 2])], axis=1)
    return pos, sh_out, second


@np.errstate(over="ignore", invalid="ignore", under="ignore")
def wgsl_interpolate(layout, lhs, rhs, t):
    t = F(t)
    return wgsl_f32(lhs, rhs, t) if layout == "f32" else wgsl_f16(lhs, rhs, t, layout == "cov")


# ---- comparison -----------------------------------------------------------------------------------------------------
def f32_same(a, b):
    """Bit for bit, every NaN equal to every NaN."""
    a, b = np.asarray(a, F), np.asarray(b, F)
    return a.shape == b.shape and bool(np.all((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))))


def half_words_same(a, b):
    """Packed half words bit for bit, every NaN half equal to every NaN half."""
    a, b = np.asarray(a, np.uint32), np.asarray(b, np.uint32)
    if a.shape != b.shape:
        return False
    ok = True
    for shift in (0, 16):
        ha, hb = (a >> shift) & 0xFFFF, (b >> shift) & 0xFFFF
        nan_a = ((ha & 0x7C00) == 0x7C00) & ((ha & 0x3FF) != 0)
        nan_b = ((hb & 0x7C00) == 0x7C00) & ((hb & 0x3FF) != 0)
        ok &= bool(np.all((ha == hb) | (nan_a & nan_b)))
    return ok


def planes_same(layout, got, want):
    if layout == "f32":
        return all(f32_same(g, w) for g, w in zip(got, want))
    return f32_same(got[0], want[0]) and half_words_same(got[1], want[1]) and half_words_same(got[2], want[2])


def assert_planes(layout, got, want, what):
    names = ("pos_vis", "sh", "rot", "scale_opacity") if layout == "f32" else ("pos_vis", "sh_packed", "second")
    for name, g, w in zip(names, got, want):
        same = f32_same(g, w) if (layout == "f32" or name == "pos_vis") else half_words_same(g, w)
        if not same:
            bad = np.flatnonzero(~np.all((np.asarray(g).view(np.uint32) == np.asarray(w).view(np.uint32)).reshape(len(g), -1), 1))
            raise AssertionError(f"{what}: {layout} {name} differs at gaussians {bad[:8].tolist()} ({len(bad)} in all)")


ALL = IC.cases()


def run_oracle(case, layout):
    t = IO.factor(case["time"], case["time_start"], case["time_stop"])
    return t, IO.interpolate(layout, case["lhs"][layout], case["rhs"][layout], t)


# ---- the oracle against the transliteration -------------------------------------------------------------------------
@pytest.mark.parametrize("layout", IC.LAYOUTS)
@pytest.mark.parametrize("case", ALL, ids=[c["name"] for c in ALL])
def test_oracle_matches_wgsl_transliteration(case, layout):
    t = IO.factor(case["time"], case["time_start"], case["time_stop"])
    assert f32_same(t, wgsl_factor(case["time"], case["time_start"], case["time_stop"]))
    got = IO.interpolate(layout, case["lhs"][layout], case["rhs"][layout], t)
    want = wgsl_interpolate(layout, case["lhs"][layout], case["rhs"][layout], t)
    assert_planes(layout, got, want, case["name"])


def test_factor_refusals():
    for args in ((np.nan, 0, 1), (0, np.inf, 1), (0, 0, -np.inf), (3e38, -3e38, 3e38)):
        with pytest.raises(ValueError):
            IO.factor(*args)
    with np.errstate(over="ignore", invalid="ignore"):
        assert np.isnan((F(3e38) - F(-3e38)) / (F(3e38) - F(-3e38)))     # (3e38 - -3e38) / inf
    assert IO.factor(3e38, -3e38, 0.0) == F(1.0)                          # (inf) / 3e38 -> clamped


def test_half_conversions_match_numpy():
    h = np.arange(1 << 16, dtype=np.uint32)
    want = h.astype(np.uint16).view(np.float16).astype(F)
    got = np.array([IO.half_to_float(x) for x in h], F)
    assert f32_same(got, want)
    rng = np.random.default_rng(0)
    f = np.concatenate([rng.integers(0, 1 << 32, 200_000, dtype=np.uint64).astype(np.uint32).view(F),
                        want, want * F(1.0004883), (want.astype(np.float64) + np.float64(2.0) ** -25).astype(F),
                        np.array([65504, 65519.99, 65520, 65536, 1e10, 2.0 ** -25, 2.0 ** -24 * 1.5, 2.0 ** -24 * 2.5], F)])
    f = f[~np.isnan(f)]
    with np.errstate(over="ignore"):
        want16 = f.astype(np.float16).view(np.uint16)
    got16 = np.array([IO.float_to_half(x) for x in f], np.uint16)
    assert np.array_equal(got16, want16)
    assert IO.float_to_half(np.nan) & 0x7C00 == 0x7C00 and IO.float_to_half(np.nan) & 0x3FF


# ---- every class is reached -----------------------------------------------------------------------------------------
def by_class():
    d = {}
    for c in ALL:
        d.setdefault(c["cls"], []).append(c)
    return d


def factor_of(c):
    return IO.factor(c["time"], c["time_start"], c["time_stop"])


def test_every_factor_class_is_reached():
    d = by_class()
    assert set(d) == set(IC.CLASSES)
    bits = lambda x: int(np.float32(x).view(np.uint32))
    assert bits(factor_of(d["t_zero"][0])) == 0 and bits(factor_of(d["t_one"][0])) == bits(1.0)
    assert sorted(float(factor_of(c)) for c in d["t_clamped"]) == [0.0, 1.0]
    assert bits(factor_of(d["t_clamped"][0])) == 0                                  # clamped to +0
    assert 0 < factor_of(d["t_interior"][0]) < 1
    eps = IC.EPS_D
    for cls, stop in (("d_at_eps", eps), ("d_below_eps", np.nextafter(eps, F(0))), ("d_above_eps", np.nextafter(eps, F(1)))):
        assert F(d[cls][0]["time_stop"]) - F(d[cls][0]["time_start"]) == stop, cls
    assert 0 < factor_of(d["d_at_eps"][0]) < 1 and 0 < factor_of(d["d_above_eps"][0]) < 1
    assert bits(factor_of(d["d_below_eps"][0])) == 0                                # below eps: time < stop -> 0
    assert d["d_negative"][0]["time_stop"] < d["d_negative"][0]["time_start"] and 0 < factor_of(d["d_negative"][0]) < 1
    assert bits(factor_of(d["t_negative_zero"][0])) == 0x80000000
    c = d["time_eq_stop"][0]
    assert c["time"] == c["time_stop"] == c["time_start"] and factor_of(c) == 1
    c = d["time_below_stop"][0]
    assert c["time"] < c["time_stop"] == c["time_start"] and bits(factor_of(c)) == 0
    t = factor_of(d["t_subnormal"][0])
    assert 0 < t < np.finfo(F).tiny


def test_factor_probe_gives_t():
    for c in ALL:
        if c["same"]:
            continue
        t = factor_of(c)
        _, (pos, *_) = run_oracle(c, "f32")
        want = t + F(0)                                   # +0 + t: t itself, except -0 -> +0
        assert np.array_equal(pos[0].view(np.uint32), np.full(4, want, F).view(np.uint32)), c["name"]


@np.errstate(over="ignore", invalid="ignore")
def test_every_lane_class_is_reached():
    d = by_class()
    c = d["lanes"][0]
    lp, rp = c["lhs"]["f32"], c["rhs"]["f32"]
    _, out = run_oracle(c, "f32")
    for k in (0, 1, 3):
        a, b, o = lp[k], rp[k], out[k]
        fin = np.isfinite(a) & np.isfinite(b)
        assert (np.signbit(a) & (a == 0)).any() and ((np.abs(a) < np.finfo(F).tiny) & (a != 0)).any()
        assert np.isinf(a).any() and np.isnan(a).any() and np.isnan(o[fin == False]).any()
        assert (np.isinf(o) & np.isinf(a) & np.isfinite(b)).any()                 # inf carried at 0 < t < 1
        big = fin & (np.abs(a) == IC.FMAX) & (np.abs(b) == IC.FMAX) & (np.sign(a) == np.sign(b))
        assert big.any() and np.isfinite(o[big]).all()   # the largest lanes do not overflow: |mix| <= max(|a|, |b|)
        sub = fin & (o != 0) & (np.abs(o) < np.finfo(F).tiny)
        assert sub.any()                                                          # subnormal results kept
    # at t = 0 (t = +0): lhs -0 against a positive rhs becomes +0; lhs -0 against -0 stays -0
    c0 = d["lanes_t_zero"][0]
    _, out0 = run_oracle(c0, "f32")
    a, b, o = c0["lhs"]["f32"][1], c0["rhs"]["f32"][1], out0[1]
    m = (a == 0) & np.signbit(a) & (b > 0) & np.isfinite(b)
    assert m.any() and not np.signbit(o[m]).any()
    m2 = (a == 0) & np.signbit(a) & (b == 0) & np.signbit(b)
    assert m2.any() and np.signbit(o[m2]).all()
    # lhs == rhs: mix(a, a, t) is not always a
    s = d["same"][0]
    assert s["lhs"] is s["rhs"]
    _, outs = run_oracle(s, "f32")
    a = s["lhs"]["f32"][1]
    fin = np.isfinite(a)
    assert (outs[1][fin] != a[fin]).any()


@np.errstate(over="ignore", invalid="ignore", under="ignore")
def test_every_quaternion_class_is_reached():
    c = by_class()["quaternions"][0]
    assert factor_of(c) == F(0.5)
    rl, rr = c["lhs"]["f32"][2], c["rhs"]["f32"][2]
    _, out = run_oracle(c, "f32")
    q = mix(rl, rr, F(0.5))
    l2 = ((q[:, 0] * q[:, 0] + q[:, 1] * q[:, 1]) + q[:, 2] * q[:, 2]) + q[:, 3] * q[:, 3]
    fallback = np.array([0, 0, 0, 1], F)
    zero = (q == 0).all(1)
    assert (zero & ~np.signbit(q).any(1)).any() and (zero & np.signbit(q).any(1)).any()     # zero and -0 lanes
    assert (~zero & (l2 == 0)).any()                                                        # squares underflow
    assert np.isinf(l2).any() and (np.isinf(l2) & np.isfinite(q).all(1) & (out[2] == 0).any(1)).any()   # overflow
    assert np.isnan(out[2]).all(1).any()                                                    # NaN
    anti = (rl == -rr).all(1) & (rl != 0).any(1)
    assert anti.sum() >= 8 and (out[2][anti] == fallback).all()                             # antipodal at t = 0.5
    assert np.array_equal(out[2][l2 <= 0], np.tile(fallback, ((l2 <= 0).sum(), 1)))


@np.errstate(over="ignore", invalid="ignore", under="ignore")
def test_every_f16_class_is_reached():
    c = by_class()["f16_halves"][0]
    assert factor_of(c) == F(0.5)
    _, out = run_oracle(c, "f16")
    wl, wr, wo = c["lhs"]["f16"][1], c["rhs"]["f16"][1], out[1]
    for shift in (0, 16):
        hl, hr, ho = ((w >> shift) & 0xFFFF for w in (wl, wr, wo))
        fl, fr = (h.astype(np.uint16).view(np.float16).astype(np.float64) for h in (hl, hr))
        exact = 0.5 * fl + 0.5 * fr                                    # the f32 result is exact here
        fo = ho.astype(np.uint16).view(np.float16).astype(np.float64)
        tie = np.isfinite(exact) & (exact != fo)
        assert (tie & ((ho & 1) == 0) & (hl == 0x3C00) & (hr == 0x3C01)).any()     # RNE tie to even, down
        assert (tie & (hl == 0x3C01) & (hr == 0x3C02) & (ho == 0x3C02)).any()      # ... and up
        assert ((hl == 0x0001) & (hr == 0x0002) & (ho == 0x0002)).any()            # subnormal halves, a tie
        assert ((hl == 0x7BFF) & (hr == 0x7BFF) & (ho == 0x7BFF)).any()            # the largest finite stays
        nan_l = ((hl & 0x7C00) == 0x7C00) & ((hl & 0x3FF) != 0)
        assert nan_l.any() and (((ho & 0x7C00) == 0x7C00) & ((ho & 0x3FF) != 0))[nan_l].all()
    # the covariance pad half: non-zero in the inputs, +0 in the output
    _, outc = run_oracle(c, "cov")
    assert ((c["lhs"]["cov"][2][:, 3] & 0xFFFF) != 0).any() and ((c["rhs"]["cov"][2][:, 3] & 0xFFFF) != 0).any()
    assert not (outc[2][:, 3] & 0xFFFF).any()
    # narrowing past the f16 range gives +-inf (from finite halves the blend never passes 65504: the encode is held to
    # numpy's above)
    assert IO.float_to_half(65520.0) == 0x7C00 and IO.float_to_half(-1e6) == 0xFC00 and IO.float_to_half(65519.0) == 0x7BFF
