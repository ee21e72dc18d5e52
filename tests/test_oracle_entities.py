"""bgs_render_entities' oracle and host checks, without a GPU: with agreeing entities the entity oracle is the scene4d
oracle bit for bit; the mixed cases put every pair of blend kinds (and 4D splats beside each) in one tile; check_entities
refuses lists whose sort settings disagree, and render_scene's checks are unchanged."""
import itertools

import numpy as np
import pytest

import bevy_gaussian_splatting_b200 as B
import entity_cases as E
from bevy_gaussian_splatting_b200 import plugin as P
from entity_oracle import entity_oracle as EO
from scene4d_oracle import scene4d_oracle as S4O

W, H = 200, 120
VIEW = B.headless_view(W, H)


def _listed(case):
    listed, settings, nc = [], [], []
    for cloud, layout, tr, st in E.entities(case):
        u = B.GaussianSplattingPlugin.cloud_uniform(st, tr, None)
        listed.append(E.oracle_entry(cloud, layout, u, st))
        settings.append(st.to_abi())
        nc.append(st.num_classes)
    return listed, settings, nc


@pytest.mark.parametrize("case", ["agree", "agree_aabb"])
def test_agreeing_entities_are_the_scene4d_oracle(case):
    listed, settings, nc = _listed(case)
    frame = B.CloudSettings(**E.CASES[case][0]).to_abi()
    want = S4O.frame(listed, VIEW.to_abi(), frame)
    got = EO.frame(listed, VIEW.to_abi(), settings, nc)
    for key in want:
        a, b = got[key], want[key]
        assert (a == b if np.isscalar(a) else np.array_equal(a.view(np.uint32) if a.dtype == np.float32 else a,
                                                             b.view(np.uint32) if b.dtype == np.float32 else b)), key


@pytest.mark.parametrize("case", ["kinds", "modes", "surfel_4d"])
def test_kinds_share_tiles(case):
    """Every pair of blend kinds present, and 4D splats beside each kind, occur inside one tile."""
    ents = E.entities(case)
    listed, settings, nc = _listed(case)
    got = EO.frame(listed, VIEW.to_abi(), settings, nc, want_image=False)
    offs = np.cumsum([0] + [len(c) for c, _, _, _ in ents])
    seg = np.searchsorted(offs, got["rank_to_id"], side="right") - 1
    # a splat's class: its blend kind, and 3 + kind for a 4D one
    cls = np.array([E.kind(st) + (3 if layout is None else 0) for _, layout, _, st in ents])[seg]
    present = set()
    r = got["tile_ranges"]
    for t in range(len(r)):
        if r[t, 1] > r[t, 0]:
            present |= set(itertools.combinations(sorted(set(cls[got["tile_entries"][r[t, 0]:r[t, 1]]].tolist())), 2))
    kinds3 = {E.kind(st) for _, layout, _, st in ents if layout is not None}
    kinds4 = {3 + E.kind(st) for _, layout, _, st in ents if layout is None}
    need = set(itertools.combinations(sorted(kinds3), 2)) | {(a, b) for a in kinds3 for b in kinds4}
    assert need and need <= present, need - present


def _ents(*settings):
    return [(None, s, None) for s in settings]


def test_check_entities():
    a = B.CloudSettings()
    assert P.check_entities(_ents(a, B.CloudSettings(aabb=True, rasterize_mode=B.RasterizeMode.Depth, num_classes=3))) is a
    with pytest.raises(ValueError, match="radix_sort_depth_bits"):
        P.check_entities(_ents(a, B.CloudSettings(radix_sort_depth_bits=B.RadixSortDepthBits.Bits16)))
    with pytest.raises(ValueError, match="sort_all"):
        P.check_entities(_ents(a, B.CloudSettings(sort_all=True)))
    with pytest.raises(ValueError):
        P.check_entities([])
    with pytest.raises(ValueError):
        P.check_entities(_ents(*[a] * 65))
    with pytest.raises(ValueError):   # render_scene keeps refusing per-entity settings
        P.check_scene_entities(_ents(a, B.CloudSettings(aabb=True)))
