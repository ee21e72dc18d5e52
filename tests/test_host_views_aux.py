"""bgs_render_views_aux without a GPU: the ctypes prototype against the header, the C call's refusals of a NULL context and
NULL arguments, and every ValueError the plugin's check_views_aux raises before any call."""
import ctypes as C
import os
import re

import pytest

import bevy_gaussian_splatting_b200 as B
from bevy_gaussian_splatting_b200 import abi
from bevy_gaussian_splatting_b200.plugin import check_views_aux

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M = B.RasterizeMode


def test_prototype_matches_the_header():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "bgs.h")).read(), flags=re.S)
    decl = re.search(r"bgs_status bgs_render_views_aux\((.*?)\);", src, flags=re.S).group(1)
    params = [p.strip() for p in decl.split(",")]
    (argtypes,) = [a for n, _, a in abi.SYMBOLS if n == "bgs_render_views_aux"]
    assert len(argtypes) == len(params) == 15
    assert params[6:8] == ["const bgs_view* views", "uint32_t v"]
    assert argtypes[6] is C.POINTER(abi.bgs_view) and argtypes[7] is C.c_uint32
    assert params[9:13] == ["const bgs_scene_depth* depths", "void* const* out_rgba", "void* const* out_depth",
                            "void* const* out_normal"]
    assert argtypes[9] is C.POINTER(abi.bgs_scene_depth)
    assert params[13:] == ["uint32_t out_format", "int out_is_device_ptr"]
    assert argtypes[13] is C.c_uint32 and argtypes[14] is C.c_int


def test_null_context_and_arguments():
    lib = abi.load()
    args = [None, None, None, None, 0, None, 0, None, None, None, None, None, abi.BGS_FORMAT_RGBA32F, 0]
    assert lib.bgs_render_views_aux(None, *args) == abi.BGS_EINVAL
    assert lib.bgs_render_views_aux(C.c_void_p(0), *args) == abi.BGS_EINVAL


class _Handle:
    """What check_views_aux reads of a cloud handle."""

    def __init__(self, temporal=False, precompute_covariance=False):
        self.temporal, self.precompute_covariance = temporal, precompute_covariance


def _views(n):
    return [B.headless_view(64, 48)] * n


def test_check_views_aux_refusals():
    ok = [(_Handle(), B.CloudSettings(), None), (_Handle(), B.CloudSettings(aabb=True, rasterize_mode=M.Classification), None)]
    assert check_views_aux(ok, _views(2)) == ok[0][1]
    assert check_views_aux(ok, _views(abi.BGS_SCENE_MAX_CLOUDS // 2)) == ok[0][1]
    # a Depth entity is drawn (each view over its own range), unlike in check_views
    depth = ok + [(_Handle(), B.CloudSettings(rasterize_mode=M.Depth), None)]
    assert check_views_aux(depth, _views(3)) == ok[0][1]
    with pytest.raises(ValueError, match="no views"):
        check_views_aux(ok, [])
    with pytest.raises(ValueError, match="segments"):
        check_views_aux(ok, _views(abi.BGS_SCENE_MAX_CLOUDS // 2 + 1))
    with pytest.raises(ValueError, match="OpticalFlow mode"):
        check_views_aux(ok + [(_Handle(), B.CloudSettings(rasterize_mode=M.OpticalFlow), None)], _views(2))
    with pytest.raises(ValueError, match="Velocity mode"):
        check_views_aux(ok + [(_Handle(), B.CloudSettings(rasterize_mode=M.Velocity), None)], _views(2))
    with pytest.raises(ValueError, match="precomputed-covariance"):
        check_views_aux(ok + [(_Handle(precompute_covariance=True), B.CloudSettings(), None)], _views(2))
    with pytest.raises(ValueError, match="Gaussian4d"):
        check_views_aux(ok + [(_Handle(temporal=True), B.CloudSettings(), None)], _views(2))
    # check_entities' own checks: no entities, too many, disagreeing sort fields
    with pytest.raises(ValueError, match="no entities"):
        check_views_aux([], _views(1))
    with pytest.raises(ValueError, match="at most"):
        check_views_aux(ok * 40, _views(1))
    with pytest.raises(ValueError, match="depth sort"):
        check_views_aux(ok + [(_Handle(), B.CloudSettings(radix_sort_depth_bits=B.RadixSortDepthBits.Bits16), None)], _views(1))
