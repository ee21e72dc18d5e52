"""Inputs and host restatements of bgs_render_shutter's tests (tests/test_host_shutter.py, tests/test_gpu_shutter.py):
include/bgs.h's pairwise sum and mean in f32, and shutters over views_cases' room mixes whose samples differ in camera
(interpolate_view between two of the room's cameras), in every entity's transform (a translation along the shutter) and
in the Gaussian4d performer's time (shutter_times around its own time)."""
from __future__ import annotations

import dataclasses

import numpy as np

import bevy_gaussian_splatting_b200 as B
import views_cases as V

F32 = np.float32


def pairwise_sum(xs):
    """sum(0, s) of the rule over the f32 arrays xs: x_a when b - a == 1, else sum(a, m) + sum(m, b), m = a + (b - a + 1) // 2,
    each addition rounded to f32."""
    def rec(a, b):
        if b - a == 1:
            return np.asarray(xs[a], F32)
        m = a + (b - a + 1) // 2
        return (rec(a, m) + rec(m, b)).astype(F32)
    return rec(0, len(xs))


def mean(xs):
    """The rule's mean: pairwise_sum(xs) / s, rounded to f32."""
    return (pairwise_sum(xs) / F32(len(xs))).astype(F32)


# the camera move of a moving shutter: from the room's front camera to one up and to the right of it
CAM_A = V._around((0.0, 1.5, 3.0), 200, 120)
CAM_B = V._around((0.35, 1.65, 2.8), 200, 120, target=(0.1, 1.45, -1.0))
MOTION = np.array([0.12, -0.05, 0.08], F32)   # every entity's travel over the shutter
SHUTTER = 0.2                                  # the performer's shutter length (its window is [-0.2, 1.1])


def sample_views(s: int, moving: bool = True) -> list:
    """s cameras of one shutter: interpolate_view(CAM_A, CAM_B, u_i) at the midpoints u_i = (i + 0.5) / s (or CAM_A s times)."""
    if not moving:
        return [CAM_A] * s
    return [B.interpolate_view(CAM_A, CAM_B, (i + 0.5) / s) for i in range(s)]


def moved(tr, u: float):
    """The CloudTransform `tr` (None: identity) translated by u MOTION."""
    m = (tr.matrix if tr is not None else np.eye(4, dtype=F32)).astype(F32).copy()
    m[:3, 3] += F32(u) * MOTION
    return B.CloudTransform(m)


def sample_entities(listed, s: int, moving: bool = True) -> list:
    """s entity lists [(cloud, layout, transform, settings)] of views_cases.entities' `listed`: sample i with every
    transform moved to u = (i + 0.5) / s - 0.5 of MOTION and each Gaussian4d entity at shutter_times(time, SHUTTER, s)[i]
    (or `listed` s times)."""
    if not moving:
        return [list(listed) for _ in range(s)]
    out = [[] for _ in range(s)]
    for cloud, layout, tr, st in listed:
        times = B.shutter_times(st.time, SHUTTER, s) if layout is None else None
        for i in range(s):
            sti = st if times is None else dataclasses.replace(st, time=float(times[i]))
            out[i].append((cloud, layout, moved(tr, (i + 0.5) / s - 0.5), sti))
    return out
