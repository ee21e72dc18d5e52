"""bgs_render_entities_many and _pick_many without a GPU: the ctypes prototypes against the header, the cap, the C calls'
refusal of a NULL context, check_entities_many and the plugin's ValueErrors before any call, and the split cases'
pieces."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
import entities_many_cases as EM
from bevy_gaussian_splatting_b200 import abi
from bevy_gaussian_splatting_b200.plugin import GaussianSplattingPlugin, check_entities, check_entities_many

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "bgs.h")


def _params(name):
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    return [p.strip() for p in re.search(rf"bgs_status {name}\((.*?)\);", src, flags=re.S).group(1).split(",")]


def test_prototypes_are_the_capped_calls():
    """Each call takes its capped twin's parameters in the same order, and abi.py declares them alike."""
    for many, capped in (("bgs_render_entities_many", "bgs_render_entities_ex"),
                         ("bgs_render_entities_pick_many", "bgs_render_entities_pick")):
        assert _params(many) == _params(capped)
        (a,) = [args for n, _, args in abi.SYMBOLS if n == many]
        (b,) = [args for n, _, args in abi.SYMBOLS if n == capped]
        assert a == b


def test_cap():
    assert abi.BGS_ENTITIES_MANY_MAX == 65536
    assert "#define BGS_ENTITIES_MANY_MAX 65536u" in open(HEADER).read()
    assert abi.BGS_SCENE_MAX_CLOUDS == 64


def test_null_context():
    lib = abi.load()
    assert lib.bgs_render_entities_many(None, None, None, None, None, 0, None, None, None, None, None, 0, 0) == abi.BGS_EINVAL
    assert lib.bgs_render_entities_pick_many(None, None, None, None, None, 0, None, None, None, None, None, 0, 0,
                                             None) == abi.BGS_EINVAL


class _Handle:
    temporal = False
    precompute_covariance = False
    n = 4


def test_check_entities_many():
    a = B.CloudSettings()
    ents = [(_Handle(), a, None)] * 65
    with pytest.raises(ValueError, match="at most 64"):
        check_entities(ents)
    assert check_entities_many(ents) is a
    assert check_entities_many([(_Handle(), a, None)] * abi.BGS_ENTITIES_MANY_MAX) is a
    with pytest.raises(ValueError, match="render_entities_many: 65537 entities, at most 65536"):
        check_entities_many([(_Handle(), a, None)] * (abi.BGS_ENTITIES_MANY_MAX + 1))
    with pytest.raises(ValueError, match="render_entities_many: no entities"):
        check_entities_many([])
    bad = ents + [(_Handle(), B.CloudSettings(sort_all=True), None)]
    with pytest.raises(ValueError, match="render_entities_many: entity 65 has sort_all"):
        check_entities_many(bad)


def test_plugin_validation_raises_before_any_call():
    p = GaussianSplattingPlugin.__new__(GaussianSplattingPlugin)   # (no context: any C call would fail)
    view = B.headless_view(8, 4)
    for call, name in ((p.render_entities_many, "render_entities_many"), (p.render_entities_pick_many, "render_entities_pick_many")):
        with pytest.raises(ValueError, match=f"^{name}: no entities"):
            call([], view)
        with pytest.raises(ValueError, match="at most 65536"):
            call([(_Handle(), B.CloudSettings(), None)] * 65537, view)
        bad = [(_Handle(), B.CloudSettings(), None)] * 100 + [
            (_Handle(), B.CloudSettings(radix_sort_depth_bits=B.RadixSortDepthBits.Bits16), None)]
        with pytest.raises(ValueError, match="entity 100 .*depth sort"):
            call(bad, view)


@pytest.mark.parametrize("n,k", [(65 * 40, 65), (257 * 33, 257), (4097 * 40, 4097), (65536 * 33, 65536)])
def test_split_pieces(n, k):
    """k non-empty contiguous pieces of [0, n) in order; sizes 1, 31, 32 and 33 among them; some piece spans several
    key-gen tiles when n allows, and cuts sit on tile and phase-2 chunk edges."""
    ps = EM.pieces(n, k, 3)
    assert len(ps) == k and all(len(x) for x in ps)
    assert np.array_equal(np.concatenate(ps), np.arange(n))
    sizes = {len(x) for x in ps}
    assert set(EM.SMALL) <= sizes
    cuts = EM.split_cuts(n, k, 3)
    if n - 33 * k >= 8 * 3 * EM.KG_TILE:
        assert max(sizes) > 2 * EM.KG_TILE
        assert any(c % EM.KG_TILE == 0 for c in cuts[1:-1])
    if n > EM.KG_CHUNK + 64:
        assert any(c % EM.KG_CHUNK == 0 for c in cuts[1:-1])
