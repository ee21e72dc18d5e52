"""Host-side particle behaviours: the reference's `ParticleBehaviors` asset (src/morph/particle.rs:349-410).

A `ParticleBehaviors` array is a numpy structured array of `PARTICLE_BEHAVIOR_DTYPE` records, 64 B each and laid out
exactly like `bgs_particle_behavior` (include/bgs.h): the pointer `bgs_particles_create` borrows.  The step itself is
libbgs's (`GaussianSplattingPlugin.step_particles`); this module only builds and holds the records.
"""
from __future__ import annotations

import numpy as np

# ParticleBehavior {indicies: [u32; 4], velocity, acceleration, jerk: [f32; 4]} (particle.rs:349-358), repr(C)
PARTICLE_BEHAVIOR_DTYPE = np.dtype([("indices", "<u4", (4,)), ("velocity", "<f4", (4,)), ("acceleration", "<f4", (4,)),
                                    ("jerk", "<f4", (4,))])
assert PARTICLE_BEHAVIOR_DTYPE.itemsize == 64

# indices[0] values at or above this (negative as the shader's i32) mark a behaviour inactive
PARTICLE_INACTIVE = np.uint32(0x80000000)


def ParticleBehaviors(n: int) -> np.ndarray:
    """n zeroed behaviours (ParticleBehavior::default(): every one active on gaussian 0, so set indices first)."""
    return np.zeros(int(n), PARTICLE_BEHAVIOR_DTYPE)


def as_particle_behaviors(behaviors) -> np.ndarray:
    """A C-contiguous (n,) array of PARTICLE_BEHAVIOR_DTYPE: the records as given, or a ValueError."""
    a = np.asarray(behaviors)
    if a.dtype != PARTICLE_BEHAVIOR_DTYPE or a.ndim != 1:
        raise ValueError("particle behaviours must be a 1-D array of PARTICLE_BEHAVIOR_DTYPE")
    return np.ascontiguousarray(a)


def random_particle_behaviors(n: int, seed: int = 0) -> np.ndarray:
    """random_particle_behaviors (particle.rs:374-410): behaviour i moves gaussian i (indices[1..3] = 0); velocity
    U(-1, 1), acceleration U(-0.01, 0.01), jerk U(-1e-4, 1e-4) in all four lanes.  Seeded (numpy Philox) instead of the
    reference's thread RNG, so a run is reproducible."""
    n = int(n)
    rng = np.random.Generator(np.random.Philox(seed))
    b = ParticleBehaviors(n)
    b["indices"][:, 0] = np.arange(n, dtype=np.uint32)
    b["velocity"] = rng.uniform(-1.0, 1.0, (n, 4)).astype(np.float32)
    b["acceleration"] = rng.uniform(-0.01, 0.01, (n, 4)).astype(np.float32)
    b["jerk"] = rng.uniform(-1e-4, 1e-4, (n, 4)).astype(np.float32)
    return b
