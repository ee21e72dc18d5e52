"""bgs_render_shutter without a GPU: the ctypes prototype against the header, the C call's refusals of a NULL context and
NULL arguments, every ValueError the plugin's check_shutter raises before any call, the pairwise mean's restatement,
shutter_times and interpolate_view."""
import ctypes as C
import dataclasses
import os
import re

import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
import shutter_cases as SH
from bevy_gaussian_splatting_b200 import abi
from bevy_gaussian_splatting_b200.plugin import check_shutter

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M = B.RasterizeMode


def test_prototype_matches_the_header():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "bgs.h")).read(), flags=re.S)
    decl = re.search(r"bgs_status bgs_render_shutter\((.*?)\);", src, flags=re.S).group(1)
    params = [" ".join(p.split()) for p in decl.split(",")]
    (argtypes,) = [a for n, _, a in abi.SYMBOLS if n == "bgs_render_shutter"]
    assert len(argtypes) == len(params) == 13
    assert params[2:4] == ["const bgs_cloud_uniform* uniforms", "const bgs_entity_settings* entities"]
    assert argtypes[2] is C.POINTER(abi.bgs_cloud_uniform) and argtypes[3] is C.POINTER(abi.bgs_entity_settings)
    assert params[6:8] == ["const bgs_view* views", "uint32_t s"]
    assert argtypes[6] is C.POINTER(abi.bgs_view) and argtypes[7] is C.c_uint32
    assert params[9:11] == ["const bgs_scene_depth* depths", "void* out_rgba"]
    assert argtypes[9] is C.POINTER(abi.bgs_scene_depth) and argtypes[10] is C.c_void_p


def test_null_context_and_arguments():
    lib = abi.load()
    args = [None, None, None, None, 0, None, 0, None, None, None, abi.BGS_FORMAT_RGBA32F, 0]
    assert lib.bgs_render_shutter(None, *args) == abi.BGS_EINVAL
    assert lib.bgs_render_shutter(C.c_void_p(0), *args) == abi.BGS_EINVAL


class _H:
    """A stand-in handle: check_shutter compares handles by identity and reads is_4d / precompute_covariance."""
    temporal = False


def test_check_shutter_refusals():
    a, b = _H(), _H()
    st = B.CloudSettings(aabb=True)
    one = [(a, st, None), (b, B.CloudSettings(), None)]
    v = B.headless_view(64, 48)
    moved = [(a, dataclasses.replace(st, time=0.4, global_opacity=0.5, global_scale=1.5), B.CloudTransform()), one[1]]
    assert check_shutter([one, moved, one], [v] * 3) == st
    assert check_shutter([one] * (abi.BGS_SCENE_MAX_CLOUDS // 2), [v] * (abi.BGS_SCENE_MAX_CLOUDS // 2)) == st
    with pytest.raises(ValueError, match="no samples"):
        check_shutter([], [])
    with pytest.raises(ValueError, match="one view per sample"):
        check_shutter([one, one], [v])
    with pytest.raises(ValueError, match="segments"):
        check_shutter([one] * (abi.BGS_SCENE_MAX_CLOUDS // 2 + 1), [v] * (abi.BGS_SCENE_MAX_CLOUDS // 2 + 1))
    with pytest.raises(ValueError, match="one frame's size"):
        check_shutter([one, one], [v, B.headless_view(64, 40)])
    with pytest.raises(ValueError, match="sample 1 has 1 entities"):
        check_shutter([one, one[:1]], [v] * 2)
    with pytest.raises(ValueError, match="another cloud"):
        check_shutter([one, [one[1], one[0]]], [v] * 2)
    with pytest.raises(ValueError, match="aabb"):
        check_shutter([one, [(a, dataclasses.replace(st, aabb=False), None), one[1]]], [v] * 2)
    with pytest.raises(ValueError, match="time_start"):
        check_shutter([one, [(a, dataclasses.replace(st, time_start=0.5), None), one[1]]], [v] * 2)
    # check_views' own checks, on sample 0: Depth and OpticalFlow entities, no entities, disagreeing sort fields
    for mode in (M.Depth, M.OpticalFlow):
        bad = [(a, B.CloudSettings(rasterize_mode=mode), None)]
        with pytest.raises(ValueError, match=f"{mode.name} mode"):
            check_shutter([bad, bad], [v] * 2)
    with pytest.raises(ValueError, match="no entities"):
        check_shutter([[]], [v])
    with pytest.raises(ValueError, match="depth sort"):
        check_shutter([one + [(a, B.CloudSettings(radix_sort_depth_bits=B.RadixSortDepthBits.Bits16), None)]], [v])


def test_pairwise_mean_restatement():
    rng = np.random.default_rng(5)
    for m in range(7):
        x = rng.uniform(-3.0, 3.0, 1000).astype(np.float32)
        x[:4] = [0.1, 1.0 / 3.0, np.float32(1e-30), 7.0]
        assert SH.mean([x] * (1 << m)).tobytes() == x.tobytes(), m
    xs = [rng.uniform(0.0, 1.0, 1000).astype(np.float32) for _ in range(3)]
    assert SH.pairwise_sum(xs).tobytes() == ((xs[0] + xs[1]) + xs[2]).tobytes()
    assert SH.mean(xs).tobytes() == (((xs[0] + xs[1]) + xs[2]) / np.float32(3)).tobytes()
    xs = [rng.uniform(0.0, 1.0, 1000).astype(np.float32) for _ in range(5)]
    assert SH.pairwise_sum(xs).tobytes() == (((xs[0] + xs[1]) + xs[2]) + (xs[3] + xs[4])).tobytes()
    # (the order matters: the left-to-right sum differs somewhere)
    xs = [rng.uniform(0.0, 1.0, 100000).astype(np.float32) for _ in range(5)]
    seq = xs[0]
    for x in xs[1:]:
        seq = seq + x
    assert SH.pairwise_sum(xs).tobytes() != seq.tobytes()


def test_shutter_times():
    t = B.shutter_times(1.0, 0.5, 4)
    assert t.dtype == np.float32 and t.tolist() == [0.8125, 0.9375, 1.0625, 1.1875]
    assert B.shutter_times(0.35, 0.2, 1).tolist() == [np.float32(0.35)]
    f = np.float32
    for time, shutter, count in ((0.35, 0.2, 3), (-0.1, 1.0 / 3.0, 7), (12.5, 0.04, 16)):
        i = np.arange(count, dtype=f)
        want = f(time) + f(shutter) * ((i + f(0.5)) / f(count) - f(0.5))
        assert B.shutter_times(time, shutter, count).tobytes() == want.astype(f).tobytes()
        mid = B.shutter_times(time, shutter, count).astype(np.float64)
        assert abs(mid.mean() - time) < 1e-5 and abs(mid[-1] - mid[0] - shutter * (count - 1) / count) < 1e-5
    with pytest.raises(ValueError):
        B.shutter_times(0.0, 1.0, 0)


def test_interpolate_view():
    a, b = SH.CAM_A, SH.CAM_B
    for u, end in ((0.0, a), (1.0, b)):
        v = B.interpolate_view(a, b, u)
        assert v.view_from_world.tobytes() == end.view_from_world.tobytes()
        assert np.asarray(v.world_position, np.float32).tobytes() == np.asarray(end.world_position, np.float32).tobytes()
        assert v.clip_from_view.tobytes() == a.clip_from_view.tobytes() and (v.width, v.height) == (a.width, a.height)
    h = B.interpolate_view(a, b, 0.5)
    mid = (np.asarray(a.world_position, np.float64) + np.asarray(b.world_position, np.float64)) / 2
    assert np.array_equal(np.asarray(h.world_position, np.float32), mid.astype(np.float32))
    # a rigid camera at the eye: an orthonormal rotation, and the eye maps to the view-space origin
    r = h.view_from_world[:3, :3].astype(np.float64)
    assert np.abs(r @ r.T - np.eye(3)).max() < 1e-6 and abs(np.linalg.det(r) - 1.0) < 1e-6
    assert np.abs(h.view_from_world.astype(np.float64) @ np.append(mid, 1.0))[:3].max() < 1e-5
    # the slerp: the rotation halfway is equally far (in angle) from both ends
    def angle(p, q):
        return np.arccos(np.clip((np.trace(p.T @ q) - 1) / 2, -1, 1))
    ra, rb = a.view_from_world[:3, :3].astype(np.float64), b.view_from_world[:3, :3].astype(np.float64)
    assert abs(angle(ra, r) - angle(r, rb)) < 1e-6 and angle(ra, rb) > 0.05
