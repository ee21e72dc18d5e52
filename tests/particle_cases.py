"""Seeded particle-behaviour cases for the step's tests (tests/test_oracle_particles.py on the CPU, tests/test_gpu_particles.py
on the H100): one builder per class of input the rule in include/bgs.h (bgs_cloud_particles_step) distinguishes.

Each case is a dict: name, cls (the class it belongs to), pos (n, 4) f32, behaviors (PARTICLE_BEHAVIOR_DTYPE records),
dts (the step sizes, applied in turn).  `cases(scale)` builds every class; `scale` multiplies the sizes of the bulk
classes so the GPU file can reach 200 000 gaussians with the same builders.
"""
from __future__ import annotations

import numpy as np

from bevy_gaussian_splatting_b200.particles import ParticleBehaviors, random_particle_behaviors

CLASSES = ("reference", "many_steps", "subnormal", "signed_zero", "non_finite", "w_crossing", "inactive",
           "carried_indices", "permuted", "count_lt_n", "count_eq_1")

REFERENCE_DTS = (1.0 / 60.0, 1.0 / 144.0, 0.0, -1.0 / 60.0, 0.5)
INACTIVE_VALUES = (0x80000000, 0xFFFFFFFF)


def positions(n: int, seed: int) -> np.ndarray:
    """The reference generator's position plane: xyz U(-20, 20), visibility 1 (planar_3d.rs:120-168)."""
    rng = np.random.default_rng(seed)
    p = np.ones((n, 4), np.float32)
    p[:, :3] = rng.uniform(-20.0, 20.0, (n, 3)).astype(np.float32)
    return p


def _case(name, cls, pos, beh, dts):
    return {"name": name, "cls": cls, "pos": np.ascontiguousarray(pos, np.float32), "behaviors": np.ascontiguousarray(beh),
            "dts": [float(np.float32(d)) for d in dts]}


def reference(n: int, dt: float, seed: int = 0):
    return _case(f"reference_dt{dt:+.5f}", "reference", positions(n, seed), random_particle_behaviors(n, seed), [dt])


def many_steps(n: int, seed: int = 1):
    rng = np.random.default_rng(seed)
    dts = rng.uniform(-0.05, 0.1, 100)
    dts[::17] = 0.0
    return _case("many_steps", "many_steps", positions(n, seed), random_particle_behaviors(n, seed), dts)


def subnormal(n: int = 4096, seed: int = 2):
    """Subnormal acceleration and jerk with odd mantissas, so 0.5f*a (and 0.5f*j) round: the WGSL order matters.
    dt around 1 keeps the products subnormal or near the normal boundary."""
    rng = np.random.default_rng(seed)
    b = random_particle_behaviors(n, seed)
    mant = (rng.integers(1, 1 << 23, (n, 4), dtype=np.uint32) | 1).astype(np.uint32)   # odd: 0.5 * x is a tie
    sign = (rng.integers(0, 2, (n, 4), dtype=np.uint32) << 31).astype(np.uint32)
    b["acceleration"] = (mant | sign).view(np.float32)
    mant2 = (rng.integers(1, 1 << 23, (n, 4), dtype=np.uint32) | 1).astype(np.uint32)
    b["jerk"] = (mant2 | sign[::-1]).view(np.float32)
    b["velocity"][: n // 2] = 0.0             # half with v = 0: dp is the subnormal terms alone
    pos = positions(n, seed)
    pos[: n // 4] = 0.0                        # ... on p = 0, so the rounded terms land in the result unabsorbed
    return _case("subnormal", "subnormal", pos, b, [1.0, 0.75, -1.5, 3.0])


def signed_zero(dt: float = 0.0):
    """p = -0 with dt = 0: p + dp is +0 unless every term of dp is -0 (with dt = +0: v, a, j all negative or -0, so
    each product is -0; with dt = -0: all positive or +0).  Every sign combination of (p, v, a, j), two steps."""
    combos = np.array(np.meshgrid(*[[0.0, -0.0]] * 4, indexing="ij")).reshape(4, -1).T   # 16 sign patterns of zeros
    mags = np.array([0.0, 1.0, 1e-3, 3.0], np.float32)
    rows_p, rows_v, rows_a, rows_j = [], [], [], []
    for m in mags:
        for sp, sv, sa, sj in combos:
            rows_p.append(np.copysign(0.0, sp))
            rows_v.append(np.copysign(m, sv))
            rows_a.append(np.copysign(m, sa))
            rows_j.append(np.copysign(m, sj))
    k = len(rows_p)
    n = (k + 3) // 4
    pad = n * 4 - k
    lane = lambda r: np.asarray(r + [0.0] * pad, np.float32).reshape(n, 4)
    b = ParticleBehaviors(n)
    b["indices"][:, 0] = np.arange(n, dtype=np.uint32)
    b["velocity"], b["acceleration"], b["jerk"] = lane(rows_v), lane(rows_a), lane(rows_j)
    return _case(f"signed_zero_dt{'-' if np.signbit(dt) else '+'}0", "signed_zero", lane(rows_p), b, [dt, dt])


def non_finite(seed: int = 4):
    """Overflow to inf (|v|, |a|, |j| near FLT_MAX with large dt), and NaN / +-inf in each of v, a, j and p."""
    specials = np.array([np.nan, np.inf, -np.inf], np.float32)
    n = 4 * len(specials) * 2 + 8
    rng = np.random.default_rng(seed)
    b = random_particle_behaviors(n, seed)
    pos = positions(n, seed)
    row = 0
    for which in ("p", "velocity", "acceleration", "jerk"):
        for s in specials:
            for lane in (0, 3):
                if which == "p":
                    pos[row, lane] = s
                else:
                    b[which][row, lane] = s
                row += 1
    big = np.float32(3.0e38)
    b["velocity"][row:row + 2] = big
    b["acceleration"][row + 2:row + 4] = -big
    b["jerk"][row + 4:row + 6] = big
    pos[row + 6:row + 8] = big * np.float32(rng.choice([-1.0, 1.0], (2, 4)))
    return _case("non_finite", "non_finite", pos, b, [4.0, 0.5])


def w_crossing(n: int = 2048, seed: int = 5):
    """Visibility lanes just below / above 0.5 with a .w velocity that carries them across (DrawMode::Selected)."""
    rng = np.random.default_rng(seed)
    b = random_particle_behaviors(n, seed)
    pos = positions(n, seed)
    pos[:, 3] = np.float32(0.5) + rng.uniform(-0.01, 0.01, n).astype(np.float32)
    pos[::7, 3] = np.float32(0.5)
    b["velocity"][:, 3] = np.where(pos[:, 3] < 0.5, 1.0, -1.0).astype(np.float32) * rng.uniform(0.5, 1.5, n).astype(np.float32)
    return _case("w_crossing", "w_crossing", pos, b, [1.0 / 60.0, 1.0 / 60.0])


def inactive(n: int = 3000, seed: int = 6):
    """Inactive indices 0x80000000 and 0xFFFFFFFF interleaved with active ones: every third behaviour is inactive."""
    b = random_particle_behaviors(n, seed)
    b["indices"][0::3, 0] = INACTIVE_VALUES[0]
    b["indices"][1::6, 0] = INACTIVE_VALUES[1]
    return _case("inactive", "inactive", positions(n, seed), b, [1.0 / 60.0, 0.5])


def carried_indices(n: int = 1000, seed: int = 7):
    rng = np.random.default_rng(seed)
    b = random_particle_behaviors(n, seed)
    b["indices"][:, 1:] = rng.integers(0, 1 << 32, (n, 3), dtype=np.uint64).astype(np.uint32)
    return _case("carried_indices", "carried_indices", positions(n, seed), b, [1.0 / 60.0, 1.0 / 144.0])


def permuted(n: int, seed: int = 8):
    """Behaviour k moves gaussian perm[k]: count = n in a random order."""
    rng = np.random.default_rng(seed)
    b = random_particle_behaviors(n, seed)
    b["indices"][:, 0] = rng.permutation(n).astype(np.uint32)
    return _case("permuted", "permuted", positions(n, seed), b, [1.0 / 60.0, -0.25])


def count_lt_n(n: int, seed: int = 9):
    """count = n / 3 behaviours over a random subset of n gaussians: the rest must stay bit-identical."""
    rng = np.random.default_rng(seed)
    count = max(1, n // 3)
    b = random_particle_behaviors(count, seed)
    b["indices"][:, 0] = rng.choice(n, count, replace=False).astype(np.uint32)
    return _case("count_lt_n", "count_lt_n", positions(n, seed), b, [1.0 / 60.0, 0.5])


def count_eq_1(n: int = 500, seed: int = 10):
    b = random_particle_behaviors(1, seed)
    b["indices"][0, 0] = n - 1                 # the last gaussian
    return _case("count_eq_1", "count_eq_1", positions(n, seed), b, [1.0 / 60.0, 1.0 / 60.0, 0.5])


def cases(scale: int = 1) -> list[dict]:
    """Every class; the bulk classes at `scale` times their CPU size."""
    n = 5000 * scale
    out = [reference(n, dt, seed=i) for i, dt in enumerate(REFERENCE_DTS)]
    out += [many_steps(2000 * scale), subnormal(), signed_zero(0.0), signed_zero(-0.0), non_finite(), w_crossing(), inactive(),
            carried_indices(), permuted(n), count_lt_n(n), count_eq_1()]
    return out


def same_bits(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """Elementwise: identical f32 bits, or both NaN (NaN compared as a class: CUDA's NaN payload is not x86's)."""
    a = np.asarray(a, np.float32)
    b = np.asarray(b, np.float32)
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


def assert_same(got: np.ndarray, want: np.ndarray, what: str):
    ok = same_bits(got, want)
    if not ok.all():
        bad = np.argwhere(~ok)[:6]
        raise AssertionError(f"{what}: {int((~ok).sum())} values differ, first at {bad.tolist()}: "
                             f"got {[got[tuple(i)] for i in bad]} want {[want[tuple(i)] for i in bad]}")


def assert_same_behaviors(got: np.ndarray, want: np.ndarray, what: str):
    assert np.array_equal(got["indices"], want["indices"]), f"{what}: indices differ"
    for f in ("velocity", "acceleration", "jerk"):
        assert_same(got[f], want[f], f"{what}: {f}")
