"""ctypes loader for the particle-step CPU oracle (particle_oracle/libparticle_oracle.so).  TEST INFRASTRUCTURE ONLY.

May be imported only by tests/ and scripts/.  See particle_oracle.h for the rule.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libparticle_oracle.so")

_lib = None


def build() -> None:
    subprocess.run(["make", "-C", _HERE, "-s"], check=True)


def load() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            build()
        lib = C.CDLL(LIB_PATH)
        lib.orc_particle_step.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_float]
        lib.orc_particle_step.restype = C.c_int
        lib.orc_particle_c6.argtypes = []
        lib.orc_particle_c6.restype = C.c_float
        _lib = lib
    return _lib


def c6() -> np.float32:
    return np.float32(load().orc_particle_c6())


def particle_step(pos_vis: np.ndarray, behaviors: np.ndarray, dt: float):
    """One step -> (new pos_vis (n, 4) f32, new behaviours).  The inputs are not modified.  ValueError for an active
    index >= n or a duplicate active index (the inputs libbgs refuses)."""
    p = np.array(pos_vis, np.float32, order="C", copy=True)
    assert p.ndim == 2 and p.shape[1] == 4
    b = np.array(behaviors, copy=True, order="C")
    assert b.dtype.itemsize == 64 and b.ndim == 1
    rc = load().orc_particle_step(p.ctypes.data_as(C.c_void_p), len(p), b.ctypes.data_as(C.c_void_p), len(b), C.c_float(dt))
    if rc != 0:
        raise ValueError("an active behaviour names a gaussian >= n, or two name the same one")
    return p, b


def particle_steps(pos_vis: np.ndarray, behaviors: np.ndarray, dts):
    """particle_step applied for each dt in turn."""
    p, b = pos_vis, behaviors
    for dt in dts:
        p, b = particle_step(p, b, dt)
    return p, b
