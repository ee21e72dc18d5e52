"""bgs_render_entities_aux without a GPU: the plugin's ValueErrors before any call, the ctypes prototype, and the C
call's argument checks that need no context."""
import ctypes as C
import os
import re

import pytest

import bevy_gaussian_splatting_b200 as B
from bevy_gaussian_splatting_b200 import abi
from bevy_gaussian_splatting_b200.plugin import check_entities_aux

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M = B.RasterizeMode


class _Handle:
    """Stands in for a resident cloud: check_entities_aux reads only these attributes."""

    def __init__(self, temporal=False, precompute_covariance=False):
        self.temporal, self.precompute_covariance = temporal, precompute_covariance


def test_plugin_refuses_what_the_aux_frames_cannot_draw():
    ok = [(_Handle(), B.CloudSettings(), None), (_Handle(), B.CloudSettings(aabb=True, rasterize_mode=M.Classification), None)]
    assert check_entities_aux(ok) == ok[0][1]
    with pytest.raises(ValueError, match="Gaussian4d"):
        check_entities_aux(ok + [(_Handle(temporal=True), B.CloudSettings(gaussian_mode=B.GaussianMode.Gaussian4d), None)])
    with pytest.raises(ValueError, match="covariance"):
        check_entities_aux(ok + [(_Handle(precompute_covariance=True), B.CloudSettings(), None)])
    with pytest.raises(ValueError, match="Velocity"):
        check_entities_aux(ok + [(_Handle(), B.CloudSettings(rasterize_mode=M.Velocity), None)])
    # render_entities' own checks come first: no entities, too many, disagreeing sort fields
    with pytest.raises(ValueError, match="no entities"):
        check_entities_aux([])
    with pytest.raises(ValueError, match="at most"):
        check_entities_aux(ok * 40)
    with pytest.raises(ValueError, match="depth sort"):
        check_entities_aux(ok + [(_Handle(), B.CloudSettings(radix_sort_depth_bits=B.RadixSortDepthBits.Bits16), None)])


def test_prototype_matches_the_header():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "bgs.h")).read(), flags=re.S)
    decl = re.search(r"bgs_status bgs_render_entities_aux\((.*?)\);", src, flags=re.S).group(1)
    params = [p.strip() for p in decl.split(",")]
    (argtypes,) = [a for n, _, a in abi.SYMBOLS if n == "bgs_render_entities_aux"]
    assert len(argtypes) == len(params) == 15
    assert params[11:13] == ["void* out_depth", "void* out_normal"]


def test_null_context_and_arguments():
    lib = abi.load()
    args = [None, None, None, None, 0, None, None, None, None, None, None, None, abi.BGS_FORMAT_RGBA32F, 0]
    assert lib.bgs_render_entities_aux(None, *args) == abi.BGS_EINVAL
    assert lib.bgs_render_entities_aux(C.c_void_p(0), *args) == abi.BGS_EINVAL
