"""The particle-step oracle (particle_oracle/) against an independent numpy float32 transliteration of
src/morph/particle.wgsl:23-53, bit for bit (NaN compared as a class), on every class of tests/particle_cases.py."""
import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
import particle_cases as PC
from particle_oracle import particle_oracle as PO

F = np.float32


def wgsl_step(pos: np.ndarray, beh: np.ndarray, dt: float):
    """particle.wgsl, line by line, in numpy float32 (every operand f32, so every operation rounds once, no FMA).
    WGSL evaluates `a * b * c` left to right; the abstract constants 0.5 and 1.0 / 6.0 become f32 where they meet
    an f32 operand."""
    pos = pos.copy()
    beh = beh.copy()
    dt = F(dt)
    idx = beh["indices"][:, 0].view(np.int32)              # `indicies: vec4<i32>` (particle.wgsl:15)
    live = idx >= 0                                         # particle.wgsl:46: `if (behavior.indicies.x < 0) { return; }`
    point = pos[np.where(live, idx, 0)]                     # particle.wgsl:31-32
    v, a, j = beh["velocity"], beh["acceleration"], beh["jerk"]
    half, sixth = F(0.5), F(1.0 / 6.0)
    # particle.wgsl:36-38
    delta_position = v * dt + half * a * dt * dt + sixth * j * dt * dt * dt
    delta_velocity = a * dt + half * j * dt * dt
    delta_acceleration = j * dt
    # particle.wgsl:40-42
    new_position = point + delta_position
    new_velocity = v + delta_velocity
    new_acceleration = a + delta_acceleration
    # particle.wgsl:50-52
    pos[idx[live]] = new_position[live]
    beh["velocity"][live] = new_velocity[live]
    beh["acceleration"][live] = new_acceleration[live]
    return pos, beh


@np.errstate(over="ignore", invalid="ignore")
def run_both(case):
    p_o, b_o = case["pos"], case["behaviors"]
    p_w, b_w = case["pos"], case["behaviors"]
    for dt in case["dts"]:
        p_o, b_o = PO.particle_step(p_o, b_o, dt)
        p_w, b_w = wgsl_step(p_w, b_w, dt)
    return (p_o, b_o), (p_w, b_w)


ALL = PC.cases()


def test_c6_is_wgsl_sixth_rounded_once():
    assert PO.c6() == F(1.0 / 6.0)
    assert PO.c6().view(np.uint32) == 0x3E2AAAAB


@pytest.mark.parametrize("case", ALL, ids=[c["name"] for c in ALL])
def test_oracle_matches_wgsl_transliteration(case):
    (p_o, b_o), (p_w, b_w) = run_both(case)
    PC.assert_same(p_o, p_w, f"{case['name']} positions")
    PC.assert_same_behaviors(b_o, b_w, case["name"])
    assert np.array_equal(b_o["jerk"].view(np.uint32), case["behaviors"]["jerk"].view(np.uint32))   # never written
    assert np.array_equal(b_o["indices"], case["behaviors"]["indices"])


def _moved(case):
    (p, b), _ = run_both(case)
    return p, b


def test_every_class_is_reached():
    by_cls = {}
    for c in ALL:
        by_cls.setdefault(c["cls"], []).append(c)
    assert set(by_cls) == set(PC.CLASSES)
    assert sorted(c["dts"][0] for c in by_cls["reference"]) == sorted(float(F(d)) for d in PC.REFERENCE_DTS)
    assert len(by_cls["many_steps"][0]["dts"]) == 100 and len(set(by_cls["many_steps"][0]["dts"])) > 50

    # subnormal: 0.5f * a rounds (the exact half is not representable) for some a, and it shows in a result
    sub = by_cls["subnormal"][0]
    a = sub["behaviors"]["acceleration"]
    assert (np.abs(a) < np.finfo(np.float32).tiny).all()
    assert ((F(0.5) * a).astype(np.float64) != a.astype(np.float64) * 0.5).any()
    p, b = _moved(sub)
    assert (b["velocity"][: len(a) // 2] != 0).any()

    # signed zeros: p = -0, dt = +-0 gives both +0 (some term +0) and -0 (every term -0)
    assert sorted(np.signbit(c["dts"][0]) for c in by_cls["signed_zero"]) == [False, True]
    for c in by_cls["signed_zero"]:
        p, _ = _moved(c)
        zeros = p[p == 0]
        assert (np.signbit(zeros)).any() and (~np.signbit(zeros)).any(), c["name"]

    # overflow to inf from finite inputs, and NaN / inf propagated from each of v, a, j, p
    nf = by_cls["non_finite"][0]
    p, b = _moved(nf)
    fin_in = np.isfinite(nf["pos"]).all(1) & np.isfinite(nf["behaviors"]["velocity"]).all(1) & \
        np.isfinite(nf["behaviors"]["acceleration"]).all(1) & np.isfinite(nf["behaviors"]["jerk"]).all(1)
    assert np.isinf(p[fin_in]).any()
    assert np.isnan(p).any() and np.isinf(p[~fin_in]).any()
    for f in ("velocity", "acceleration", "jerk"):
        assert (~np.isfinite(nf["behaviors"][f])).any()
    assert (~np.isfinite(nf["pos"])).any()

    # .w crossing 0.5 both ways
    wc = by_cls["w_crossing"][0]
    p, _ = _moved(wc)
    w0, w1 = wc["pos"][:, 3], p[:, 3]
    assert ((w0 < 0.5) & (w1 >= 0.5)).any() and ((w0 >= 0.5) & (w1 < 0.5)).any()

    # inactive: both values, interleaved with active ones; their gaussians and records are untouched
    ina = by_cls["inactive"][0]
    ix = ina["behaviors"]["indices"][:, 0]
    assert set(PC.INACTIVE_VALUES) <= set(ix.tolist()) and (ix < 0x80000000).sum() > 0
    p, b = _moved(ina)
    off = ix >= 0x80000000
    assert np.array_equal(b["velocity"][off], ina["behaviors"]["velocity"][off])
    named = np.zeros(len(ina["pos"]), bool)
    named[ix[~off]] = True
    assert np.array_equal(p[~named], ina["pos"][~named]) and not np.array_equal(p[named], ina["pos"][named])

    assert (by_cls["carried_indices"][0]["behaviors"]["indices"][:, 1:] != 0).all(1).any()
    per = by_cls["permuted"][0]["behaviors"]["indices"][:, 0]
    assert sorted(per.tolist()) == list(range(len(per))) and (per != np.arange(len(per))).any()
    lt = by_cls["count_lt_n"][0]
    assert 1 < len(lt["behaviors"]) < len(lt["pos"])
    p, _ = _moved(lt)
    named = np.zeros(len(lt["pos"]), bool)
    named[lt["behaviors"]["indices"][:, 0]] = True
    assert np.array_equal(p[~named].view(np.uint32), lt["pos"][~named].view(np.uint32))
    assert len(by_cls["count_eq_1"][0]["behaviors"]) == 1
    assert any(len(c["behaviors"]) == len(c["pos"]) for c in ALL)


def test_oracle_refuses_what_libbgs_refuses():
    pos = PC.positions(10, 0)
    b = B.random_particle_behaviors(3, 0)
    b["indices"][2, 0] = 10
    with pytest.raises(ValueError):
        PO.particle_step(pos, b, 0.1)
    b["indices"][2, 0] = 1                     # duplicates behaviour 1
    with pytest.raises(ValueError):
        PO.particle_step(pos, b, 0.1)
    b["indices"][2, 0] = 0xFFFFFFFF            # inactive: not a duplicate, not out of range
    PO.particle_step(pos, b, 0.1)


def test_random_particle_behaviors_distributions():
    b = B.random_particle_behaviors(200_000, 3)
    assert b.dtype.itemsize == 64 and b.dtype == B.PARTICLE_BEHAVIOR_DTYPE
    assert np.array_equal(b["indices"][:, 0], np.arange(200_000)) and not b["indices"][:, 1:].any()
    for f, r in (("velocity", 1.0), ("acceleration", 0.01), ("jerk", 1e-4)):
        x = b[f]
        assert x.min() >= -r and x.max() < r and x.min() < -0.99 * r and x.max() > 0.99 * r, f
        assert abs(float(x.mean())) < 0.01 * r, f
    assert np.array_equal(B.random_particle_behaviors(1000, 3), B.random_particle_behaviors(1000, 3))
    assert not np.array_equal(B.random_particle_behaviors(1000, 3), B.random_particle_behaviors(1000, 4))
